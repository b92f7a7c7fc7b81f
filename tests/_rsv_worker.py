"""One rank of a test world for ReduceScatterv.  Usage as _worker.py: _rsv_worker.py <scenario>
--out FILE [scenario args] -mpi-* flags.  The scenarios drive the product through the public
mpi_b200 API / C ABI and compare every rank's block bit for bit with the rank-order reduction of the
C oracle (_rsv_ref.py); the rest (argument parsing, Init, result file) is _worker.py's."""
import ctypes
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _rsv_ref as V  # noqa: E402
import _worker as W  # noqa: E402
from _footprint_worker import LAYOUTS, OPS, Guarded, Run, check, epv, gen_values, layout_offsets, mode_for  # noqa: E402
from _worker import DTYPES, L, O, SEED, check_equal, free_buffer, make_buffer, read_buffer, mpi  # noqa: E402

OPNAMES = {o[0]: (o[1], o[2]) for o in OPS}


def sentinel(dt, count):
    return np.full(count, -7, dtype=dt)


def ctable(counts):
    return (ctypes.c_size_t * len(counts))(*counts)


def same_bytes(a, b, opname):
    """Byte for byte, except the payload of a NaN that a SUM made from two NaNs: which operand's payload
    an add propagates depends on how the compiler ordered the operands of that add (H100: the vector
    and the scalar loop of two kernels may differ), so there only both being NaN is required.  MAX and
    MIN select an operand and must match exactly."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.size != b.size:
        return False
    if a.size == 0:
        return True
    differ = (a.view(np.uint8).reshape(a.size, -1) != b.view(np.uint8).reshape(b.size, -1)).any(axis=1)
    if opname == "sum" and a.dtype.kind == "f":
        differ &= ~(np.isnan(a) & np.isnan(b))
    return not differ.any()


def indivisible(n, dt):
    """A length no world size divides evenly, whose balanced blocks start at different residues mod 16."""
    return 1000 * n * epv(dt) + n // 2 + 1 if n > 1 else 1001


def tables(n, dt):
    """(name, table): uniform at the Scan tests' counts, a balanced split of an indivisible length,
    zero entries (rank 1 has none) and one rank holding most of the data."""
    out = [("uniform %d" % c, [c] * n) for c in (0, 1, 3, 4, 5, 255, 256, 257, 4096, 65537)]
    out.append(("balanced", V.balanced(indivisible(n, dt), n)))
    out.append(("zeros", [0 if r % 3 == 1 else 37 * r + 5 for r in range(n)]))
    out.append(("skewed", V.skewed(70001, n)))
    return out


def run_rsv(kind, ins, counts, op, inplace, null_recv=False):
    """One ReduceScatterv; returns what this rank's block holds afterwards.  In place the recv is this
    rank's block of send.  null_recv: the C ABI with a NULL recv (this rank's count is 0)."""
    rank = mpi.Rank()
    d = V.displs(counts)
    dt = ins[rank].dtype
    send = make_buffer(kind, ins[rank])
    if null_recv:
        sp = send.ptr if kind == "heap" else (send.ctypes.data if send.size else None)
        rc = L.load().b200mpi_reduce_scatterv(sp, None, ctable(counts), O.NP2DT[np.dtype(dt)], op, L.DEVICE if kind == "heap" else L.HOST)
        assert rc == 0, L.last_error()
        got = np.zeros(0, dtype=dt)
    else:
        recv = send[d[rank]:d[rank + 1]] if inplace else make_buffer(kind, sentinel(dt, counts[rank]))
        out, learnt = mpi.ReduceScatterv(send, recv, counts, op)
        assert learnt == counts and out is recv, (learnt, counts)
        got = np.array(read_buffer(recv), copy=True)
        if not inplace:
            free_buffer(recv)
    whole = np.array(read_buffer(send), copy=True)
    if inplace:  # the rest of send is untouched
        check_equal(np.concatenate([whole[:d[rank]], whole[d[rank + 1]:]]),
                    np.concatenate([ins[rank][:d[rank]], ins[rank][d[rank + 1]:]]), "in place: send outside the block untouched")
    else:
        check_equal(whole, ins[rank], "send untouched")
    free_buffer(send)
    return got


def check_table(kind, dn, name, counts, opname, inplace, salt):
    """One table against the oracle; a uniform one also against ReduceScatter of the same inputs."""
    rank, n = mpi.Rank(), mpi.Size()
    dt = DTYPES[dn]
    op, oop = OPNAMES[opname]
    ins = gen_values(dt, n, sum(counts), salt)
    what = "%s table=%s op=%s kind=%s inplace=%s rank=%d n=%d" % (dn, name, opname, kind, inplace, rank, n)
    null_recv = counts[rank] == 0 and not inplace and salt % 2 == 0
    got = run_rsv(kind, ins, counts, op, inplace, null_recv)
    W.trace("reduce_scatterv " + what)
    assert same_bytes(got, V.rsv_oracle(ins, counts, oop, rank), opname), "reduce_scatterv against the oracle " + what
    if name.startswith("uniform") and counts[0]:
        src, out = make_buffer(kind, ins[rank]), make_buffer(kind, sentinel(dt, counts[0]))
        L.load().b200mpi_set_algo(L.COLL_REDUCE_SCATTER, L.ALGO_TWOSHOT)  # the rank-order form, not the switch's
        mpi.ReduceScatter(src, out, op)
        L.load().b200mpi_set_algo(L.COLL_REDUCE_SCATTER, 0)
        rs = np.array(read_buffer(out))
        assert same_bytes(got, rs, opname), "reduce_scatterv == reduce_scatter byte for byte " + what
        free_buffer(out)
        free_buffer(src)
    return 1


def scenario_rsv(a):
    """Every dtype and op over the tables, with the memory kind and in/out of place rotating over the
    tables so that each combination meets every dtype and op; then a table learnt from len(recv)."""
    rank, n = mpi.Rank(), mpi.Size()
    kinds = a.kinds.split(",")
    done, salt = 0, 0
    for di, dn in enumerate(a.dtypes.split(",")):
        for oi, (opname, _, _) in enumerate(OPS):
            for ti, (name, counts) in enumerate(tables(n, DTYPES[dn])):
                i = ti + oi + di
                salt += 1
                done += check_table(kinds[i % len(kinds)], dn, name, counts, opname, (i // len(kinds)) % 2 == 1, salt)
    counts = V.balanced(indivisible(n, np.float64), n)
    ins = gen_values(np.float64, n, sum(counts), 4242)
    recv, learnt = mpi.ReduceScatterv(np.array(ins[rank]), np.empty(counts[rank], np.float64), None, mpi.MAX)
    assert learnt == counts, (learnt, counts)
    check_equal(recv, V.rsv_oracle(ins, counts, O.MAX, rank), "reduce_scatterv with a learnt table")
    done += 1
    mpi.Barrier()
    return {"checked": done}


def do_footprint(R, dn, counts, layout, opname, inplace, kind):
    """One guarded call: only recv is written, with the oracle's block; an out-of-place send and every
    guard stay byte-identical; in place, send equals its input with this rank's block replaced."""
    lib, rank, n = R.lib, R.rank, R.n
    dt = DTYPES[dn]
    op, oop = OPNAMES[opname]
    call = R.next_call("reduce_scatterv")
    offs = layout_offsets(layout, dt, n, call)
    d = V.displs(counts)
    mine = counts[rank]
    ins = gen_values(dt, n, d[-1], call)
    send = Guarded(kind, dt, d[-1], offs[rank][0], rank, call, body=ins[rank])
    recv = None
    if inplace:  # recv == send + displacement of this rank's block
        sub = send.sub(d[rank], d[rank + 1])
        rp = sub.ptr if kind == "heap" else sub.ctypes.data
    elif mine:
        recv = Guarded(kind, dt, mine, offs[rank][1], rank, call + 1)
        rp = recv.ptr()
    else:
        rp = None  # count 0: NULL recv
    mk = L.DEVICE if kind == "heap" else L.HOST
    rc = lib.b200mpi_reduce_scatterv(send.ptr(), rp, ctable(counts), O.NP2DT[np.dtype(dt)], op, mk)
    what = R.what("reduce_scatterv", L.ALGO_TWOSHOT, dt, opname, d[-1], layout, offs, kind, inplace) + " table=%s" % counts
    assert rc == 0, (what, rc, L.last_error())
    want = V.rsv_oracle(ins, counts, oop, rank)
    blocks = [x[d[rank]:d[rank + 1]] for x in ins]
    mode = mode_for(opname, dt, O.ORDER_RANK)
    if inplace:
        send.set_body(want, lo=d[rank])
        check(send, what + " [in-place send]", mode if mine else "exact", blocks, lo=d[rank])
    else:
        check(send, what + " [send must be unchanged]")
        if recv is not None:
            recv.set_body(want)
            check(recv, what + " [recv]", mode, blocks)
            recv.free()
    send.free()


def scenario_rsv_footprint(a):
    """Guarded views at the four layouts of _footprint_worker.py, with its special values, over a
    uniform, a balanced, a zero-entry and a skewed table."""
    R = Run(types.SimpleNamespace(trim="full"))
    n = R.n
    for di, dn in enumerate(("f32", "f64", "i64")):
        dt = DTYPES[dn]
        e = epv(dt)
        tabs = [[4 * e + 1] * n, V.balanced(n * 9 * e + 1, n), [0 if r % 2 else 3 * e + r for r in range(n)], V.skewed(4097, n)]
        for ti, counts in enumerate(tabs):
            for li, layout in enumerate(LAYOUTS):
                i = ti + li + di
                inplace = layout in ("aligned", "mixed") and (ti + di) % 2 == 1
                kind = R.kind_for(i, sum(counts) * dt().itemsize)
                do_footprint(R, dn, counts, layout, OPS[i % 3][0], inplace, kind)
    mpi.Barrier()
    return {"checked": sum(R.done.values())}


def scenario_rsv_mismatch(a):
    """Ranks that disagree (a table that differs in one entry or by a swap, op, dtype, or a rank calling
    ReduceScatter against ReduceScatterv with a uniform table) get B200MPI_ERR_PEER on every rank with
    send and recv untouched; the next ReduceScatterv works."""
    rank, n = mpi.Rank(), mpi.Size()
    lib = L.load()
    odd = rank == 1
    base = [1000 + 3 * r for r in range(n)]
    one = list(base)
    one[0] += 1 if odd else 0
    swap = list(base)
    if odd:
        swap[0], swap[1] = swap[1], swap[0]
    half = [c // 2 for c in base]
    uni = [1000] * n
    cases = (
        ("table differs in one entry", lambda s, r: lib.b200mpi_reduce_scatterv(s, r, ctable(one), L.F32, L.SUM, mk)),
        ("tables differ by a swap", lambda s, r: lib.b200mpi_reduce_scatterv(s, r, ctable(swap), L.F32, L.SUM, mk)),
        ("different op", lambda s, r: lib.b200mpi_reduce_scatterv(s, r, ctable(base), L.F32, L.MAX if odd else L.SUM, mk)),
        ("different dtype", lambda s, r: lib.b200mpi_reduce_scatterv(s, r, ctable(half), L.I64 if odd else L.F64, L.MIN, mk)),
        ("reduce_scatter against reduce_scatterv", lambda s, r: lib.b200mpi_reduce_scatter(s, r, 1000, L.F32, L.SUM, mk) if odd
         else lib.b200mpi_reduce_scatterv(s, r, ctable(uni), L.F32, L.SUM, mk)),
    )
    total = sum(base) + n
    xs = [np.arange(total, dtype=np.float32) * (r + 1) - 300 for r in range(n)]
    done = 0
    for kind in ("heap", "host"):
        mk = L.DEVICE if kind == "heap" else L.HOST
        x = make_buffer(kind, xs[rank])
        y = make_buffer(kind, sentinel(np.float32, 2 * max(base)))
        xp = x.ptr if kind == "heap" else x.ctypes.data
        yp = y.ptr if kind == "heap" else y.ctypes.data
        for name, call in cases:
            # a successful call first leaves its result in the staging block
            assert lib.b200mpi_reduce_scatterv(xp, yp, ctable(base), L.F32, L.SUM, mk) == 0, L.last_error()
            sends = [v[:sum(base)] for v in xs]
            check_equal(np.array(read_buffer(y))[:base[rank]], V.rsv_oracle(sends, base, O.SUM, rank), "before %s (%s)" % (name, kind))
            if kind == "heap":
                y.copy_from_host(sentinel(np.float32, 2 * max(base)))
            else:
                y[:] = sentinel(np.float32, 2 * max(base))
            rc = call(xp, yp)
            assert rc == L.ERR_PEER, (name, kind, rc, L.last_error())
            check_equal(np.array(read_buffer(y)), sentinel(np.float32, 2 * max(base)), "%s %s: recv untouched" % (name, kind))
            check_equal(np.array(read_buffer(x)), xs[rank], "%s %s: send untouched" % (name, kind))
            done += 1
        # and the world still works
        assert lib.b200mpi_reduce_scatterv(xp, yp, ctable(base), L.F32, L.MAX, mk) == 0, L.last_error()
        check_equal(np.array(read_buffer(y))[:base[rank]], V.rsv_oracle([v[:sum(base)] for v in xs], base, O.MAX, rank), "after mismatches (%s)" % kind)
        free_buffer(x)
        free_buffer(y)
        done += 1
    mpi.Barrier()
    return {"checked": done}


def scenario_rsv_wrap(a):
    """ReduceScatterv call after call across the scrub that ends on epoch 0 (the world starts a few
    launches below it).  Reports the epoch before and after."""
    n = mpi.Size()
    first = L.get_param("epoch")
    done = 0
    for i in range(12):
        dn = ("f32", "f64", "i64")[i % 3]
        name, counts = (("balanced", V.balanced(indivisible(n, DTYPES[dn]), n)), ("skewed", V.skewed(65537, n)),
                        ("uniform 257", [257] * n))[i % 3]
        kind = "host" if i % 4 == 3 else "heap"
        done += check_table(kind, dn, name, counts, OPS[i % 3][0], i % 2 == 1, 900 + 2 * i + 1)
    mpi.Barrier()
    return {"checked": done, "epoch_first": first, "epoch_last": L.get_param("epoch")}


def scenario_rsv_sharded_allreduce(a):
    """The owner-computes Allreduce: displacements from an i64 Exscan of each rank's count, an in-place
    ReduceScatterv and then an in-place Allgatherv over the same buffer and table equal a two-shot
    Allreduce of the same inputs bit for bit, on a balanced split of an indivisible count and on a
    skewed table, heap and host."""
    rank, n = mpi.Rank(), mpi.Size()
    lib = L.load()
    done = 0
    for ti, dn in enumerate(("f32", "f64", "i64")):
        dt = DTYPES[dn]
        for counts in (V.balanced(indivisible(n, dt), n), V.skewed(100003, n)):
            mine = np.array([counts[rank]], dtype=np.int64)
            displ = np.zeros(1, dtype=np.int64)  # rank 0's Exscan recv is not written: its displacement stays 0
            mpi.Exscan(mine, displ, mpi.SUM)
            d = int(displ[0])
            assert d == sum(counts[:rank]), (d, counts)
            opname = OPS[(ti + len(counts)) % 3][0]
            op = OPNAMES[opname][0]
            ins = gen_values(dt, n, sum(counts), 7000 + 10 * ti + counts[-1] % 7)
            lib.b200mpi_set_algo(L.COLL_ALLREDUCE, L.ALGO_TWOSHOT)
            src, ref = make_buffer("heap", ins[rank]), make_buffer("heap", sentinel(dt, sum(counts)))
            mpi.Allreduce(src, ref, op)
            want = ref.to_host()
            free_buffer(ref)
            free_buffer(src)
            lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
            for kind in ("heap", "host"):
                buf = make_buffer(kind, ins[rank])
                mpi.ReduceScatterv(buf, buf[d:d + counts[rank]], counts, op)
                mpi.Allgatherv(buf[d:d + counts[rank]], buf, counts)
                got = np.array(read_buffer(buf))
                assert same_bytes(got, want, opname), "sharded allreduce != two-shot allreduce (%s %s %s table=%s)" % (dn, opname, kind, counts)
                free_buffer(buf)
                done += 1
    mpi.Barrier()
    return {"checked": done}


def scenario_rsv_large(a):
    """64 MiB per rank on a skewed table: an f32 SUM and an i64 MAX, each rank's block checked block by
    block against the oracle."""
    rank, n = mpi.Rank(), mpi.Size()
    block = 1 << 20
    for dt, op, oop in ((np.float32, mpi.SUM, O.SUM), (np.int64, mpi.MAX, O.MAX)):
        total = (64 << 20) // np.dtype(dt).itemsize
        counts = V.skewed(total, n, heavy=1)
        d = V.displs(counts)
        send = mpi.Alloc(total, dt).copy_from_host(O.fill(dt, SEED + rank, total))
        recv = mpi.Alloc(counts[rank], dt).copy_from_host(sentinel(dt, counts[rank]))
        mpi.ReduceScatterv(send, recv, counts, op)
        got = recv.to_host()
        for lo in range(d[rank], d[rank + 1], block):
            k = min(block, d[rank + 1] - lo)
            ins = [O.fill_at(dt, SEED + r, lo, k) for r in range(n)]
            check_equal(got[lo - d[rank]:lo - d[rank] + k], O.allreduce(ins, op=oop, order=O.ORDER_RANK), "large %s block at %d" % (np.dtype(dt).name, lo))
        send.free()
        recv.free()
    mpi.Barrier()
    return {"checked": 2}


def scenario_rsv_control_only(a):
    """Control plane only: ReduceScatterv refuses with B200MPI_ERR_NO_DEVICE, through the C ABI and the facade."""
    lib = L.load()
    n = mpi.Size()
    x, y = np.zeros(4 * n, dtype=np.float32), np.zeros(4, dtype=np.float32)
    rc = lib.b200mpi_reduce_scatterv(x.ctypes.data, y.ctypes.data, ctable([4] * n), L.F32, L.SUM, L.HOST)
    assert rc == L.ERR_NO_DEVICE, rc
    for call in (lambda: mpi.ReduceScatterv(x, y, [4] * n), lambda: mpi.ReduceScatterv(x, y)):
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
