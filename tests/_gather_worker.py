"""One rank of a test world for Gather, Scatter, Gatherv, Scatterv and Allgatherv.  Usage as
_worker.py: _gather_worker.py <scenario> --out FILE [scenario args] -mpi-* flags.  The scenarios drive
the product through the public mpi_b200 API / C ABI and check every result against the CPU oracle
(_gather_oracle.py, test infrastructure only); the rest (argument parsing, Init, result file) is
_worker.py's."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _gather_oracle as G  # noqa: E402
import _worker as W  # noqa: E402
from _worker import L, O, SEED, check_equal, free_buffer, make_buffer, mpi, read_buffer  # noqa: E402


GDTYPES = {"u8": np.uint8, "f32": np.float32, "f64": np.float64, "i64": np.int64}


def gfill(dt, seed, count):
    if np.dtype(dt) == np.uint8:
        return np.frombuffer(O.fill(np.int64, seed, count // 8 + 1).tobytes(), dtype=np.uint8)[:count].copy()
    return O.fill(dt, seed, count)


def sentinel(dt, count):
    return np.full(count, 0xA5 if np.dtype(dt) == np.uint8 else -7, dtype=dt)


def check_rooted(kind, dt, counts, root, with_all=True):
    """Gather(v) and Scatter(v) to / from `root`, and Allgatherv, with the table `counts`, out of place
    and in place, bit-exact against the oracle.  The fixed-count entries run when the table is
    uniform.  Non-root recv sentinels and every send buffer must stay untouched.  Returns calls checked."""
    rank, n = mpi.Rank(), mpi.Size()
    displ = [0]
    for c in counts:
        displ.append(displ[-1] + c)
    total, mine = displ[-1], counts[rank]
    uniform = len(set(counts)) == 1
    what = "%s %s counts=%s root=%d" % (kind, np.dtype(dt).name, counts if len(set(counts)) > 1 else "%dx%d" % (n, counts[0]), root)
    ins = [gfill(dt, SEED + 17 * r + total, counts[r]) for r in range(n)]
    packed = G.gatherv(ins)
    big = gfill(dt, SEED + 5 + total, total)  # root's send of the scatter
    done = 0
    for inplace in (False, True):
        own = inplace and rank == root
        # Gather(v)
        if own:
            arr = sentinel(dt, total)
            arr[displ[root]:displ[root + 1]] = ins[root]
            recv = make_buffer(kind, arr)
            send = recv[displ[root]:displ[root + 1]]
        else:
            recv = make_buffer(kind, sentinel(dt, total))
            send = make_buffer(kind, ins[rank])
        if uniform:
            mpi.Gather(send, recv, root)
        else:
            mpi.Gatherv(send, recv, root, counts)
        if rank == root:
            check_equal(read_buffer(recv), packed, "gather %s inplace=%s" % (what, inplace))
        else:
            check_equal(read_buffer(recv), sentinel(dt, total), "gather %s: non-root recv untouched" % what)
        if not own:
            check_equal(read_buffer(send), ins[rank], "gather %s: send untouched" % what)
            free_buffer(send)
        free_buffer(recv)
        # Scatter(v)
        send = make_buffer(kind, big) if rank == root else None
        recv = send[displ[root]:displ[root + 1]] if own else make_buffer(kind, sentinel(dt, mine))
        if uniform:
            got = mpi.Scatter(send, recv, root)
        else:
            got, _ = mpi.Scatterv(send, recv, counts, root)
        check_equal(read_buffer(got), G.scatterv(big, counts, rank), "scatter %s inplace=%s" % (what, inplace))
        if rank == root:
            check_equal(read_buffer(send), big, "scatter %s: root send untouched" % what)
            free_buffer(send)
        if not own:
            free_buffer(recv)
        done += 2
        # Allgatherv
        if with_all:
            if inplace:
                arr = sentinel(dt, total)
                arr[displ[rank]:displ[rank + 1]] = ins[rank]
                recv = make_buffer(kind, arr)
                send = recv[displ[rank]:displ[rank + 1]]
            else:
                recv = make_buffer(kind, sentinel(dt, total))
                send = make_buffer(kind, ins[rank])
            got, _ = mpi.Allgatherv(send, recv, counts)
            check_equal(read_buffer(got), packed, "allgatherv %s inplace=%s" % (what, inplace))
            if not inplace:
                check_equal(read_buffer(send), ins[rank], "allgatherv %s: send untouched" % what)
                free_buffer(send)
            free_buffer(recv)
            done += 1
    return done


def scenario_gather(a):
    """Gather / Scatter / Allgatherv with uniform counts over every root, every dtype, heap and host."""
    n = mpi.Size()
    done = 0
    for kind in a.kinds.split(","):
        for dn in a.dtypes.split(","):
            for count in [int(s) for s in a.sizes.split(",")]:
                for root in range(n):
                    done += check_rooted(kind, GDTYPES[dn], [count] * n, root, with_all=root == 0)
    mpi.Barrier()
    return {"checked": done}


def v_tables(n):
    """Tables with zero entries, odd counts (displacements misaligned for every access width), a single
    non-empty rank and one rank carrying most of the data."""
    return [
        [0] * n,
        [2 * r + 3 for r in range(n)],
        [0 if r % 2 == 0 else 4 * r + 1 for r in range(n)],
        [1001 if r == n - 1 else 0 for r in range(n)],
        [70001 if r == n // 2 else 5 + r for r in range(n)],
        [16 * (r + 1) for r in range(n)][::-1],
    ]


def scenario_gatherv(a):
    n = mpi.Size()
    done = 0
    for kind in a.kinds.split(","):
        for dn in a.dtypes.split(","):
            for counts in v_tables(n):
                for root in range(n):
                    done += check_rooted(kind, GDTYPES[dn], counts, root, with_all=root == 0)
    mpi.Barrier()
    return {"checked": done}


def scenario_gather_unaligned(a):
    """Heap offsets that are not 16-byte aligned and differ between ranks: odd element offsets for
    bytes, 4/8-byte offsets for the wider types, and 16-byte sizes at 8/16/24-byte offsets (ranks
    then pick different access widths for the same call)."""
    rank, n = mpi.Rank(), mpi.Size()
    done = 0
    for dn, dt in GDTYPES.items():
        for counts in ([1003] * n, [2 * r + 999 for r in range(n)], [4096] * n):
            displ = [0]
            for c in counts:
                displ.append(displ[-1] + c)
            total = displ[-1]
            ins = [gfill(dt, SEED + 3 * r + total, counts[r]) for r in range(n)]
            so, ro = 1 + rank % 3, 1 + (rank + 1) % 2
            sbig, rbig = mpi.Alloc(total + 8, dt), mpi.Alloc(total + 8, dt)
            for root in sorted({0, n - 1}):
                send = sbig[so:so + counts[rank]].copy_from_host(ins[rank])
                recv = rbig[ro:ro + total].copy_from_host(sentinel(dt, total))
                mpi.Gatherv(send, recv, root, counts)
                check_equal(recv.to_host(), G.gatherv(ins) if rank == root else sentinel(dt, total), "unaligned gatherv %s root=%d" % (dn, root))
                whole = G.gatherv(ins)
                src = sbig[so:so + total].copy_from_host(whole) if rank == root else None
                out = rbig[ro:ro + counts[rank]]
                mpi.Scatterv(src, out, counts, root)
                check_equal(out.to_host(), G.scatterv(whole, counts, rank), "unaligned scatterv %s root=%d" % (dn, root))
                done += 2
            ag = rbig[ro:ro + total]
            mpi.Allgatherv(sbig[so:so + counts[rank]].copy_from_host(ins[rank]), ag, counts)
            check_equal(ag.to_host(), G.gatherv(ins), "unaligned allgatherv %s" % dn)
            done += 1
            sbig.free()
            rbig.free()
    mpi.Barrier()
    return {"checked": done}


def scenario_gather_mismatch(a):
    """Tables that differ by a swap of two counts or in one entry, and ranks that disagree on root:
    B200MPI_ERR_PEER on every rank, buffers untouched (heap and host), and the next Gather works."""
    import ctypes
    rank, n = mpi.Rank(), mpi.Size()
    lib = L.load()
    base = [3 + 5 * r for r in range(n)]
    swapped = list(base)
    swapped[0], swapped[1] = swapped[1], swapped[0]
    one_off = list(base)
    one_off[n - 1] += 1
    cap = sum(base) + 64
    done = 0
    for kind in ("heap", "host"):
        x = make_buffer(kind, gfill(np.float32, SEED + rank, cap))
        y = make_buffer(kind, sentinel(np.float32, cap))
        xp = x.ptr if kind == "heap" else x.ctypes.data
        yp = y.ptr if kind == "heap" else y.ctypes.data
        mk = L.DEVICE if kind == "heap" else L.HOST
        for other in (swapped, one_off):
            table = other if rank == 1 else base
            tab = (ctypes.c_size_t * n)(*table)
            calls = (("gatherv", lambda: lib.b200mpi_gatherv(xp, yp, tab, L.F32, 0, mk)),
                     ("scatterv", lambda: lib.b200mpi_scatterv(xp, yp, tab, L.F32, 0, mk)),
                     ("allgatherv", lambda: lib.b200mpi_allgatherv(xp, yp, tab, L.F32, mk)))
            for name, call in calls:
                rc = call()
                assert rc == L.ERR_PEER, (name, kind, table, rc, L.last_error())
                check_equal(read_buffer(y), sentinel(np.float32, cap), "%s %s table %s: recv untouched" % (name, kind, table))
                check_equal(read_buffer(x), gfill(np.float32, SEED + rank, cap), "%s %s: send untouched" % (name, kind))
                done += 1
        # ranks that disagree on root
        for name, fn in (("gather", lib.b200mpi_gather), ("scatter", lib.b200mpi_scatter)):
            rc = fn(xp, yp, 5, L.F32, rank % 2, mk)
            assert rc == L.ERR_PEER, (name, kind, rc, L.last_error())
            check_equal(read_buffer(y), sentinel(np.float32, cap), "%s %s root disagreement: recv untouched" % (name, kind))
            done += 1
        # and the world still works
        ins = [gfill(np.float32, SEED + r, 5) for r in range(n)]
        mpi.Gather(make_buffer(kind, ins[rank]), y[:5 * n], 0)
        if rank == 0:
            check_equal(read_buffer(y)[:5 * n], G.gatherv(ins), "gather after mismatches (%s)" % kind)
        free_buffer(x)
        free_buffer(y)
        done += 1
    mpi.Barrier()
    return {"checked": done}


def scenario_gather_strings(a):
    """helloworld's strings, a different length on every rank: Allgatherv and Gatherv with the counts
    learnt from the lengths; the receiver splits the packed bytes with the returned counts."""
    rank, n = mpi.Rank(), mpi.Size()
    words = ['"Hello from node %d%s"' % (r, "!" * (3 * r)) for r in range(n)]
    done = 0
    got, counts = mpi.Allgatherv(words[rank])
    assert counts == [len(w.encode()) for w in words], counts
    parts, lo = [], 0
    for c in counts:
        parts.append(got[lo:lo + c].tobytes().decode())
        lo += c
    assert parts == words, parts
    done += 1
    for root in range(n):
        got, counts = mpi.Gatherv(words[rank], None, root)
        if rank == root:
            assert got.tobytes().decode() == "".join(words), got
        else:
            assert got is None
        done += 1
    # a recv that is too small is replaced, one that is larger is used through a view
    got, _ = mpi.Allgatherv(words[rank], np.zeros(2, dtype=np.uint8))
    assert got.tobytes().decode() == "".join(words)
    big = np.full(4096, 7, dtype=np.uint8)
    got, _ = mpi.Allgatherv(words[rank], big)
    assert got.size == sum(counts) and got.tobytes().decode() == "".join(words) and big[sum(counts)] == 7
    # Scatterv: the other ranks learn their block length from root
    whole = np.frombuffer("".join(words).encode(), dtype=np.uint8).copy()
    table = [len(w.encode()) for w in words] if rank == 0 else None
    got, counts = mpi.Scatterv(whole if rank == 0 else None, np.empty(0, dtype=np.uint8), table, 0)
    assert got.tobytes().decode() == words[rank], got
    done += 3
    mpi.Barrier()
    return {"checked": done}


def scenario_gather_fullsize(a):
    """Gather of f32 16 Mi elements per rank (64 MiB each), bit-exact, then Scatter it back."""
    rank, n = mpi.Rank(), mpi.Size()
    count = 1 << 24
    send = mpi.Alloc(count, np.float32).copy_from_host(O.fill(np.float32, SEED + rank, count))
    recv = mpi.Alloc(count * n, np.float32) if rank == 0 else None
    mpi.Gather(send, recv, 0)
    if rank == 0:
        got = recv.to_host()
        for r in range(n):
            check_equal(got[r * count:(r + 1) * count], O.fill(np.float32, SEED + r, count), "gather f32 16Mi block %d" % r)
    back = mpi.Alloc(count, np.float32)
    mpi.Scatter(recv, back, 0)
    check_equal(back.to_host(), O.fill(np.float32, SEED + rank, count), "scatter(gather(x)) == x")
    for b in (send, recv, back):
        if b is not None:
            b.free()
    mpi.Barrier()
    return {"checked": 2}


def scenario_gather_control_only(a):
    """Control plane only: the new entries refuse with B200MPI_ERR_NO_DEVICE, through the C ABI and the facade."""
    import ctypes
    n = mpi.Size()
    lib = L.load()
    x = np.zeros(4 * n, dtype=np.float32)
    tab = (ctypes.c_size_t * n)(*([4] * n))
    rcs = [lib.b200mpi_gather(x.ctypes.data, x.ctypes.data, 4, L.F32, 0, L.HOST),
           lib.b200mpi_scatter(x.ctypes.data, x.ctypes.data, 4, L.F32, 0, L.HOST),
           lib.b200mpi_gatherv(x.ctypes.data, x.ctypes.data, tab, L.F32, 0, L.HOST),
           lib.b200mpi_scatterv(x.ctypes.data, x.ctypes.data, tab, L.F32, 0, L.HOST),
           lib.b200mpi_allgatherv(x.ctypes.data, x.ctypes.data, tab, L.F32, L.HOST)]
    assert rcs == [L.ERR_NO_DEVICE] * 5, rcs
    for call in (lambda: mpi.Gather(x[:4], x, 0), lambda: mpi.Scatter(x, x[:4], 0), lambda: mpi.Gatherv(x[:4], x, 0, [4] * n),
                 lambda: mpi.Scatterv(x, x[:4], [4] * n, 0), lambda: mpi.Allgatherv(x[:4], x, [4] * n), lambda: mpi.Allgatherv(x[:4])):
        try:
            call()
            raise AssertionError("data call succeeded without a device")
        except mpi.MpiError as e:
            if e.code != L.ERR_NO_DEVICE:
                raise
    return {"checked": 11}


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_")})

if __name__ == "__main__":
    W.main()
