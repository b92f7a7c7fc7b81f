"""One rank of a test world for Scan and Exscan.  Usage as _worker.py: _scan_worker.py <scenario>
--out FILE [scenario args] -mpi-* flags.  The scenarios drive the product through the public
mpi_b200 API / C ABI and compare every rank's result bit for bit with the rank-order prefix of the
C oracle (_scan_ref.py); the rest (argument parsing, Init, result file) is _worker.py's."""
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _scan_ref as S  # noqa: E402
import _worker as W  # noqa: E402
from _footprint_worker import LAYOUTS, OPS, Guarded, Run, check, counts_for, epv, gen_values, layout_offsets, mode_for  # noqa: E402
from _worker import DTYPES, L, O, SEED, check_equal, free_buffer, make_buffer, read_buffer, mpi  # noqa: E402

OPNAMES = {o[0]: (o[1], o[2]) for o in OPS}


def sentinel(dt, count):
    return np.full(count, -7, dtype=dt)


def scan_passes(n, dt):
    """Vectors per world message at which scan_kernel's grid gains a CTA (b200mpi.cu: launch_scan)."""
    u = {2: 8 if np.dtype(dt).itemsize == 4 else 4, 4: 4, 8: 2}.get(n, 1)
    return [n * 512 * u]


def run_scan(kind, ins, op, exclusive, inplace):
    """One Scan or Exscan through the facade; returns what this rank's recv holds afterwards."""
    rank = mpi.Rank()
    dt = ins[rank].dtype
    send = make_buffer(kind, ins[rank])
    recv = send if inplace else make_buffer(kind, sentinel(dt, ins[rank].size))
    (mpi.Exscan if exclusive else mpi.Scan)(send, recv, op)
    got = np.array(read_buffer(recv), copy=True)
    if not inplace:
        check_equal(read_buffer(send), ins[rank], "send untouched")
        free_buffer(recv)
    free_buffer(send)
    return got


def check_pair(kind, dn, count, opname, inplace, salt):
    """Scan and Exscan of the same inputs: each against the oracle prefix, Scan on rank n-1 against a
    two-shot Allreduce, and Scan == combine(Exscan, x_r) on ranks >= 1."""
    rank, n = mpi.Rank(), mpi.Size()
    dt = DTYPES[dn]
    op, oop = OPNAMES[opname]
    ins = gen_values(dt, n, count, salt)
    what = "%s count=%d op=%s kind=%s inplace=%s rank=%d n=%d" % (dn, count, opname, kind, inplace, rank, n)
    scan = run_scan(kind, ins, op, False, inplace)
    check_equal(scan, S.scan_oracle(ins, oop, rank), "scan " + what)
    ex = run_scan(kind, ins, op, True, inplace)
    want = S.scan_oracle(ins, oop, rank, exclusive=True)
    # rank 0 of an Exscan keeps its recv: the sentinel out of place, its own input in place
    check_equal(ex, want if want is not None else (ins[0] if inplace else sentinel(dt, count)), "exscan " + what)
    if rank >= 1:
        check_equal(scan, S.apply(oop, ex, ins[rank]), "scan == combine(exscan, x_r) " + what)
    if n > 1:
        L.load().b200mpi_set_algo(L.COLL_ALLREDUCE, L.ALGO_TWOSHOT)
        src, out = make_buffer("heap", ins[rank]), make_buffer("heap", sentinel(dt, count))
        mpi.Allreduce(src, out, op)
        if rank == n - 1:
            check_equal(scan, out.to_host(), "scan on rank n-1 == two-shot allreduce " + what)
        free_buffer(out)
        free_buffer(src)
        L.load().b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
    return 2


def scenario_scan(a):
    """Every dtype and op over the --sizes counts, with the memory kind and in/out of place rotating
    over the counts so that each combination meets every dtype and op; then one count that spans many
    4 KiB ownership blocks per rank."""
    n = mpi.Size()
    kinds = a.kinds.split(",")
    sizes = [int(s) for s in a.sizes.split(",")]
    done, salt = 0, 0
    for di, dn in enumerate(a.dtypes.split(",")):
        for oi, (opname, _, _) in enumerate(OPS):
            for ci, count in enumerate(sizes):
                i = ci + oi + di
                salt += 1
                done += check_pair(kinds[i % len(kinds)], dn, count, opname, (i // len(kinds)) % 2 == 1, salt)
    lib = L.load()
    old = L.get_param("own_block_bytes")
    lib.b200mpi_set_param(b"own_block_bytes", 4096)
    for di, dn in enumerate(a.dtypes.split(",")):
        count = (n * 25 * 256 + 100) * epv(DTYPES[dn]) + 1
        for oi, (opname, _, _) in enumerate(OPS):
            salt += 1
            done += check_pair("heap", dn, count, opname, (oi + di) % 2 == 1, salt)
    lib.b200mpi_set_param(b"own_block_bytes", old)
    if n == 1:  # a world of one: Exscan with a NULL recv writes nothing and succeeds
        x = np.arange(5, dtype=np.float64)
        assert lib.b200mpi_exscan(x.ctypes.data, None, 5, L.F64, L.SUM, L.HOST) == 0, L.last_error()
        done += 1
    mpi.Barrier()
    return {"checked": done}


def do_footprint(R, dn, count, layout, opname, inplace, kind, exclusive, null_recv=False):
    """One guarded call: only recv is written, with the oracle prefix; Exscan leaves rank 0's recv,
    and every guard, byte-identical."""
    lib, rank, n = R.lib, R.rank, R.n
    dt = DTYPES[dn]
    op, oop = OPNAMES[opname]
    coll = "exscan" if exclusive else "scan"
    call = R.next_call(coll)
    offs = layout_offsets(layout, dt, n, call)
    if inplace:
        offs = [(s, s) for s, _ in offs]
    ins = gen_values(dt, n, count, call)
    send = Guarded(kind, dt, count, offs[rank][0], rank, call, body=ins[rank])
    recv = send if inplace else None if null_recv else Guarded(kind, dt, count, offs[rank][1], rank, call + 1)
    mk = L.DEVICE if kind == "heap" else L.HOST
    fn = lib.b200mpi_exscan if exclusive else lib.b200mpi_scan
    rc = fn(send.ptr(), recv.ptr() if recv is not None else None, count, O.NP2DT[np.dtype(dt)], op, mk)
    what = R.what(coll, L.ALGO_TWOSHOT, dt, opname, count, layout, offs, kind, inplace)
    assert rc == 0, (what, rc, L.last_error())
    want = S.scan_oracle(ins, oop, rank, exclusive)
    if want is None:
        if recv is not None:
            check(recv, what + " [exscan rank 0 recv must not be written]")
    else:
        recv.set_body(want)
        check(recv, what + " [recv]", mode_for(opname, dt, O.ORDER_RANK), ins[:rank + 1])
    if not inplace:
        check(send, what + " [send must be unchanged]")
        if recv is not None:
            recv.free()
    send.free()


def scenario_scan_footprint(a):
    """Guarded views at the four layouts of _footprint_worker.py, with its special values."""
    R = Run(types.SimpleNamespace(trim="full"))
    n = R.n
    for di, dn in enumerate(("f32", "f64", "i64")):
        dt = DTYPES[dn]
        for ci, count in enumerate(counts_for(dt, scan_passes(n, dt), R.trim)):
            for li, layout in enumerate(LAYOUTS):
                i = ci + li + di
                inplace = layout in ("aligned", "mixed") and ci % 2 == 1
                kind = R.kind_for(i, count * dt().itemsize)
                for exclusive in (False, True):
                    do_footprint(R, dn, count, layout, OPS[i % 3][0], inplace, kind, exclusive)
    # Exscan with a NULL recv on rank 0, heap and host
    for kind in ("heap", "host"):
        do_footprint(R, "f64", 4097, "mixed", "sum", False, kind, True, null_recv=R.rank == 0)
    mpi.Barrier()
    return {"checked": sum(R.done.values())}


def scenario_scan_mismatch(a):
    """Ranks that disagree (Scan against Exscan, either against Allreduce, op, count, dtype) get
    B200MPI_ERR_PEER on every rank with send and recv untouched; the next Scan works."""
    rank, n = mpi.Rank(), mpi.Size()
    lib = L.load()
    c = 1000
    odd = rank == 1
    old_ll = L.get_param("ll_max_bytes")
    assert lib.b200mpi_set_param(b"ll_max_bytes", 0) == 0  # the LL Allreduce carries no signature
    cases = (
        ("scan against exscan", lambda s, r: (lib.b200mpi_exscan if odd else lib.b200mpi_scan)(s, r, c, L.F32, L.SUM, mk)),
        ("scan against allreduce", lambda s, r: (lib.b200mpi_allreduce if odd else lib.b200mpi_scan)(s, r, c, L.F32, L.SUM, mk)),
        ("exscan against allreduce", lambda s, r: (lib.b200mpi_allreduce if odd else lib.b200mpi_exscan)(s, r, c, L.F32, L.SUM, mk)),
        ("different op", lambda s, r: lib.b200mpi_scan(s, r, c, L.F32, L.MAX if odd else L.SUM, mk)),
        ("different count", lambda s, r: lib.b200mpi_exscan(s, r, c - 1 if odd else c, L.F32, L.SUM, mk)),
        ("different dtype", lambda s, r: lib.b200mpi_scan(s, r, c // 2, L.I64 if odd else L.F64, L.MIN, mk)),
    )
    done = 0
    for kind in ("heap", "host"):
        mk = L.DEVICE if kind == "heap" else L.HOST
        xs = [np.arange(c, dtype=np.float32) * (r + 1) - 300 for r in range(n)]
        x = make_buffer(kind, xs[rank])
        y = make_buffer(kind, sentinel(np.float32, c))
        xp = x.ptr if kind == "heap" else x.ctypes.data
        yp = y.ptr if kind == "heap" else y.ctypes.data
        for name, call in cases:
            # a successful call of the same size first leaves its result in the staging block
            assert lib.b200mpi_scan(xp, yp, c, L.F32, L.SUM, mk) == 0, L.last_error()
            check_equal(np.array(read_buffer(y)), S.scan_oracle(xs, O.SUM, rank), "scan before %s (%s)" % (name, kind))
            if kind == "heap":
                y.copy_from_host(sentinel(np.float32, c))
            else:
                y[:] = sentinel(np.float32, c)
            rc = call(xp, yp)
            assert rc == L.ERR_PEER, (name, kind, rc, L.last_error())
            check_equal(np.array(read_buffer(y)), sentinel(np.float32, c), "%s %s: recv untouched" % (name, kind))
            check_equal(np.array(read_buffer(x)), xs[rank], "%s %s: send untouched" % (name, kind))
            done += 1
        # and the world still works
        assert lib.b200mpi_exscan(xp, yp, c, L.F32, L.MAX, mk) == 0, L.last_error()
        want = S.scan_oracle(xs, O.MAX, rank, exclusive=True)
        check_equal(np.array(read_buffer(y)), want if want is not None else sentinel(np.float32, c), "exscan after mismatches (%s)" % kind)
        free_buffer(x)
        free_buffer(y)
        done += 1
    assert lib.b200mpi_set_param(b"ll_max_bytes", old_ll) == 0
    mpi.Barrier()
    return {"checked": done}


def scenario_scan_wrap(a):
    """Scan and Exscan call after call across the scrub that ends on epoch 0 (the world starts a
    few launches below it).  Reports the epoch before and after."""
    rank, n = mpi.Rank(), mpi.Size()
    first = L.get_param("epoch")
    done = 0
    for i in range(12):
        dn = ("f32", "f64", "i64")[i % 3]
        count = (257, 4099, 65537)[i % 3]
        kind = "host" if i % 4 == 3 else "heap"
        done += check_pair(kind, dn, count, OPS[i % 3][0], i % 2 == 1, 900 + i)
    mpi.Barrier()
    return {"checked": done, "epoch_first": first, "epoch_last": L.get_param("epoch")}


def scenario_scan_large(a):
    """64 MiB per rank: an f32 SUM Scan and an i64 Exscan, checked block by block against the oracle."""
    rank, n = mpi.Rank(), mpi.Size()
    count, block = 16 << 20, 1 << 20
    for dt, op, exclusive in ((np.float32, mpi.SUM, False), (np.int64, mpi.SUM, True)):
        total = count if dt == np.float32 else count // 2
        send = mpi.Alloc(total, dt).copy_from_host(O.fill(dt, SEED + rank, total))
        recv = mpi.Alloc(total, dt).copy_from_host(sentinel(dt, total))
        (mpi.Exscan if exclusive else mpi.Scan)(send, recv, op)
        got = recv.to_host()
        for lo in range(0, total, block):
            k = min(block, total - lo)
            ins = [O.fill_at(dt, SEED + r, lo, k) for r in range(n)]
            want = S.scan_oracle(ins, O.SUM, rank, exclusive)
            check_equal(got[lo:lo + k], want if want is not None else sentinel(dt, k), "large %s block at %d" % (np.dtype(dt).name, lo))
        send.free()
        recv.free()
    mpi.Barrier()
    return {"checked": 2}


def scenario_scan_displacements(a):
    """The use that motivates Exscan: every rank learns its offset in a buffer packed in rank order
    from an i64 Exscan of its element count, writes its block there and completes the buffer with an
    in-place Allgatherv; every rank checks the whole buffer."""
    rank, n = mpi.Rank(), mpi.Size()
    counts = [3 + 1000 * ((7 * r) % 5) + r for r in range(n)]
    blocks = [O.fill(np.float64, SEED + 77 * r, counts[r]) for r in range(n)]
    mine = np.array([counts[rank]], dtype=np.int64)
    displ = np.zeros(1, dtype=np.int64)  # rank 0's Exscan recv is not written: its displacement stays 0
    mpi.Exscan(mine, displ, mpi.SUM)
    d = int(displ[0])
    assert d == sum(counts[:rank]), (d, counts)
    last = np.empty(1, dtype=np.int64)
    mpi.Scan(mine, last, mpi.SUM)
    assert int(last[0]) == d + counts[rank]
    for kind in ("heap", "host"):
        total = sum(counts)
        if kind == "heap":
            out = mpi.Alloc(total, np.float64).copy_from_host(sentinel(np.float64, total))
            out[d:d + counts[rank]].copy_from_host(blocks[rank])
        else:
            out = sentinel(np.float64, total)
            out[d:d + counts[rank]] = blocks[rank]
        got, learnt = mpi.Allgatherv(out[d:d + counts[rank]], out)
        assert learnt == counts, learnt
        check_equal(np.array(read_buffer(got)), np.concatenate(blocks), "allgatherv at exscan displacements (%s)" % kind)
        free_buffer(out)
    mpi.Barrier()
    return {"checked": 3}


def scenario_scan_control_only(a):
    """Control plane only: Scan and Exscan refuse with B200MPI_ERR_NO_DEVICE, through the C ABI and the facade."""
    lib = L.load()
    x, y = np.zeros(4, dtype=np.float32), np.zeros(4, dtype=np.float32)
    for fn in (lib.b200mpi_scan, lib.b200mpi_exscan):
        rc = fn(x.ctypes.data, y.ctypes.data, 4, L.F32, L.SUM, L.HOST)
        assert rc == L.ERR_NO_DEVICE, rc
    for call in (lambda: mpi.Scan(x, y), lambda: mpi.Exscan(x, y), lambda: mpi.Exscan(x, None)):
        try:
            call()
            raise AssertionError("data call succeeded without a device")
        except mpi.MpiError as e:
            if e.code != L.ERR_NO_DEVICE:
                raise
    return {"checked": 5}


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_")})

if __name__ == "__main__":
    W.main()
