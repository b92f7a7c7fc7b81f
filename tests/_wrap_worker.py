"""One rank of a test world that drives the 32-bit counters across their wraps.  Usage as _worker.py:
_wrap_worker.py <scenario> --out FILE [--family F --variants V --boundary B] -mpi-* flags.

Worlds start near a boundary through the test hooks B200MPI_EPOCH_START / B200MPI_LL_SEQ_START and
walk onto it with b200mpi_barrier() calls, one stride each.  Every result is compared with the oracle
(oracle/, _gather_oracle.py, _alltoallv_ref.py); the rest (argument parsing, Init, result file) is
_worker.py's.

The launch whose end value is 0 (start 2^32 - 4095, epoch index 2^20 - 1) is always scrub_kernel:
2^20 - 1 is scrub_every - 1 modulo every allowed scrub period.  So each collective runs at the last
launch before that scrub (start 2^32 - 8191) and at the first launch after it (start 1, whose start,
mid and end barriers compare against flag words written before the wrap)."""
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _alltoallv_ref as A  # noqa: E402
import _gather_oracle as G  # noqa: E402
import _worker as W  # noqa: E402
from _gather_worker import GDTYPES, gfill, sentinel  # noqa: E402
from _worker import ALGOS, L, O, SEED, check_equal, expect_allreduce, free_buffer, make_buffer, mpi, read_buffer  # noqa: E402

STRIDE = 4096
M32 = 1 << 32
SCRUB_EVERY = int(os.environ.get("B200MPI_SCRUB_EVERY", "16384"))


def param(name):
    v = ctypes.c_int64()
    if L.load().b200mpi_get_param(name.encode(), ctypes.byref(v)):
        raise RuntimeError(L.last_error())
    return v.value


def index_of(start):
    return (start % M32) // STRIDE


def scrub_due(start):
    return (index_of(start) & (SCRUB_EVERY - 1)) == SCRUB_EVERY - 1


def next_start():
    """The start value the next collective gets (after the scrub next_comm may insert)."""
    e = param("epoch")
    return (e + STRIDE) % M32 if scrub_due(e) else e


def place(target):
    """Burn barriers until the next collective gets start value `target`.  A miss fails."""
    for _ in range(64):
        s = next_start()
        if s == target:
            return
        if ((target - s) % M32) >= (1 << 31):
            raise AssertionError("placement overshot: next start %d, target %d" % (s, target))
        mpi.Barrier()
    raise AssertionError("placement did not reach %d (epoch %d)" % (target, param("epoch")))


def expect_epoch(want, what):
    got = param("epoch")
    if got != want % M32:
        raise AssertionError("%s: epoch %d, expected %d" % (what, got, want % M32))


# ------------------------------------------------------------------------------------------------
# One call of a family, checked against the oracle.  `v` is (dtype name, memory kind, count, in place).
def call_allreduce(algo, v, salt):
    lib = L.load()
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, inplace = v
    dt = W.DTYPES[dn]
    ins = W.inputs_for(dt, n, count, salt=salt)
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
    used = lib.b200mpi_get_algo(L.COLL_ALLREDUCE, count, O.NP2DT[np.dtype(dt)])
    if used != ALGOS[algo]:
        raise AssertionError("allreduce %s resolved to algorithm %d" % (algo, used))
    send = make_buffer(kind, ins[rank])
    recv = send if inplace else make_buffer(kind, np.zeros(count, dtype=dt))
    mpi.Allreduce(send, recv, mpi.SUM)
    want, _ = expect_allreduce(ins, O.SUM, used, n, count, dt)
    check_equal(read_buffer(recv), want, "allreduce %s %s %s count=%d inplace=%s" % (algo, dn, kind, count, inplace))
    if not inplace:
        check_equal(read_buffer(send), ins[rank], "allreduce %s: send untouched" % algo)
        free_buffer(recv)
    free_buffer(send)
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)


def call_bcast(algo, v, salt):
    lib = L.load()
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = GDTYPES[dn]
    root = (salt + 1) % n
    x = gfill(dt, SEED + salt, count)
    lib.b200mpi_set_algo(L.COLL_BCAST, ALGOS[algo])
    buf = make_buffer(kind, x if rank == root else sentinel(dt, count))
    mpi.Bcast(buf, root)
    check_equal(read_buffer(buf), x, "bcast %s %s %s count=%d root=%d" % (algo, dn, kind, count, root))
    free_buffer(buf)
    lib.b200mpi_set_algo(L.COLL_BCAST, 0)


def call_allgather(algo, v, salt):
    lib = L.load()
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = GDTYPES[dn]
    ins = [gfill(dt, SEED + salt + 7 * r, count) for r in range(n)]
    lib.b200mpi_set_algo(L.COLL_ALLGATHER, ALGOS[algo])
    send = make_buffer(kind, ins[rank])
    recv = make_buffer(kind, sentinel(dt, count * n))
    mpi.Allgather(send, recv)
    check_equal(read_buffer(recv), np.concatenate(ins), "allgather %s %s %s count=%d" % (algo, dn, kind, count))
    check_equal(read_buffer(send), ins[rank], "allgather: send untouched")
    free_buffer(send)
    free_buffer(recv)
    lib.b200mpi_set_algo(L.COLL_ALLGATHER, 0)


def call_reduce_scatter(v, salt):
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = W.DTYPES[dn]
    ins = W.inputs_for(dt, n, count * n, salt=salt)
    send = make_buffer(kind, ins[rank])
    recv = make_buffer(kind, np.zeros(count, dtype=dt))
    mpi.ReduceScatter(send, recv, mpi.SUM)
    check_equal(read_buffer(recv), O.reduce_scatter(ins, rank), "reduce_scatter %s %s count=%d" % (dn, kind, count))
    check_equal(read_buffer(send), ins[rank], "reduce_scatter: send untouched")
    free_buffer(send)
    free_buffer(recv)


def call_reduce(v, salt):
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = W.DTYPES[dn]
    root = n - 1
    ins = W.inputs_for(dt, n, count, salt=salt)
    send = make_buffer(kind, ins[rank])
    recv = make_buffer(kind, np.full(count, -7, dtype=dt))
    mpi.Reduce(send, recv, mpi.SUM, root)
    want = O.allreduce(ins) if rank == root else np.full(count, -7, dtype=dt)
    check_equal(read_buffer(recv), want, "reduce %s %s count=%d root=%d" % (dn, kind, count, root))
    check_equal(read_buffer(send), ins[rank], "reduce: send untouched")
    free_buffer(send)
    free_buffer(recv)


def call_alltoall(v, salt):
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = W.DTYPES[dn]
    ins = W.inputs_for(dt, n, count * n, salt=salt)
    send = make_buffer(kind, ins[rank])
    recv = make_buffer(kind, np.full(count * n, -1, dtype=dt))
    mpi.Alltoall(send, recv)
    check_equal(read_buffer(recv), O.alltoall(ins, rank), "alltoall %s %s count=%d" % (dn, kind, count))
    check_equal(read_buffer(send), ins[rank], "alltoall: send untouched")
    free_buffer(send)
    free_buffer(recv)


def skewed(n, count):
    """One rank carries most of the data, one sends nothing, the others odd counts."""
    return [count if r == n // 2 else (0 if r == 0 else 2 * r + 1) for r in range(n)]


def call_gatherv(v, salt):
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = GDTYPES[dn]
    counts, root = skewed(n, count), n - 1
    ins = [gfill(dt, SEED + salt + 3 * r, counts[r]) for r in range(n)]
    send = make_buffer(kind, ins[rank])
    recv = make_buffer(kind, sentinel(dt, sum(counts)))
    mpi.Gatherv(send, recv, root, counts)
    want = G.gatherv(ins) if rank == root else sentinel(dt, sum(counts))
    check_equal(read_buffer(recv), want, "gatherv %s %s counts=%s" % (dn, kind, counts))
    check_equal(read_buffer(send), ins[rank], "gatherv: send untouched")
    free_buffer(send)
    free_buffer(recv)


def call_scatterv(v, salt):
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = GDTYPES[dn]
    counts, root = skewed(n, count), 1 % n
    big = gfill(dt, SEED + salt, sum(counts))
    send = make_buffer(kind, big) if rank == root else None
    recv = make_buffer(kind, sentinel(dt, counts[rank]))
    # the C ABI, not the facade: mpi.Scatterv first broadcasts root's table, a second launch
    ptr = lambda b: b.ptr if isinstance(b, mpi.DeviceSlice) else b.ctypes.data  # noqa: E731
    rc = L.load().b200mpi_scatterv(ptr(send) if send is not None else None, ptr(recv), (ctypes.c_size_t * n)(*counts), O.NP2DT[np.dtype(dt)], root,
                                   L.DEVICE if kind == "heap" else L.HOST)
    if rc:
        raise AssertionError("scatterv: %d %s" % (rc, L.last_error()))
    check_equal(read_buffer(recv), G.scatterv(big, counts, rank), "scatterv %s %s counts=%s" % (dn, kind, counts))
    if rank == root:
        check_equal(read_buffer(send), big, "scatterv: root send untouched")
        free_buffer(send)
    free_buffer(recv)


def call_allgatherv(v, salt):
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = GDTYPES[dn]
    counts = skewed(n, count)
    ins = [gfill(dt, SEED + salt + 5 * r, counts[r]) for r in range(n)]
    send = make_buffer(kind, ins[rank])
    recv = make_buffer(kind, sentinel(dt, sum(counts)))
    got, _ = mpi.Allgatherv(send, recv, counts)
    check_equal(read_buffer(got), G.gatherv(ins), "allgatherv %s %s counts=%s" % (dn, kind, counts))
    check_equal(read_buffer(send), ins[rank], "allgatherv: send untouched")
    free_buffer(send)
    free_buffer(recv)


def call_alltoallv(v, salt):
    rank, n = mpi.Rank(), mpi.Size()
    dn, kind, count, _ = v
    dt = GDTYPES[dn]
    m = [[count if j == (i + 1) % n else 2 * i + j + 1 for j in range(n)] for i in range(n)]
    sends = [gfill(dt, SEED + salt + 31 * i, sum(m[i])) for i in range(n)]
    send = make_buffer(kind, sends[rank])
    recv = make_buffer(kind, sentinel(dt, sum(A.col(m, rank))))
    got, _ = mpi.Alltoallv(send, A.row(m, rank), recv, A.col(m, rank))
    check_equal(read_buffer(got), A.alltoallv(sends, m, rank), "alltoallv %s %s" % (dn, kind))
    check_equal(read_buffer(send), sends[rank], "alltoallv: send untouched")
    free_buffer(send)
    free_buffer(recv)


def call_barrier(v, salt):
    mpi.Barrier()


FAMILIES = {
    "oneshot": lambda v, s: call_allreduce("oneshot", v, s),
    "twoshot": lambda v, s: call_allreduce("twoshot", v, s),
    "smem": lambda v, s: call_allreduce("smem", v, s),
    "ring": lambda v, s: call_allreduce("ring", v, s),
    "bcast_oneshot": lambda v, s: call_bcast("oneshot", v, s),
    "bcast_twoshot": lambda v, s: call_bcast("twoshot", v, s),
    "allgather_push": lambda v, s: call_allgather("oneshot", v, s),
    "allgather_ring": lambda v, s: call_allgather("ring", v, s),
    "reduce_scatter": call_reduce_scatter,
    "reduce": call_reduce,
    "alltoall": call_alltoall,
    "gatherv": call_gatherv,
    "scatterv": call_scatterv,
    "allgatherv": call_allgatherv,
    "alltoallv": call_alltoallv,
    "barrier": call_barrier,
}


def parse_variants(s):
    """'f32:heap:257:in,i64:host:1001:out' -> [(dtype, kind, count, in place)]"""
    out = []
    for item in s.split(","):
        dn, kind, count, place_ = item.split(":")
        out.append((dn, kind, int(count), place_ == "in"))
    return out


def scenario_wrap_family(a):
    """The variants of one family run on the launches just before the scrub of epoch index B - 1
    (B = --boundary, 2^20 by default: that scrub's end value is 0) and again on the launches just
    after it, each one launch.  B = 2^17 puts the ring step counters (epoch * 8) across their wrap."""
    lib = L.load()
    fam = FAMILIES[X.family]
    variants = parse_variants(X.variants)
    b = int(X.boundary)
    if len(variants) > SCRUB_EVERY - 1:
        raise AssertionError("more variants than launches between two scrubs")
    if X.max_blocks:
        lib.b200mpi_set_max_blocks(int(X.max_blocks))
    first = ((b - 1 - len(variants)) * STRIDE + 1) % M32
    place(first)
    if b % (1 << 20) == 0:
        assert next_start() == (M32 - (len(variants) + 1) * STRIDE + 1) % M32
    done = 0
    for k, v in enumerate(variants):
        if next_start() != (first + k * STRIDE) % M32:
            raise AssertionError("before %s: next start %d, expected %d" % (X.family, next_start(), (first + k * STRIDE) % M32))
        fam(v, k)
        done += 1
    # the scrub of index b - 1 comes next, then the first launch after the boundary
    assert scrub_due(param("epoch")), "the scrub of index %d is not due" % (b - 1)
    if b % (1 << 20) == 0:
        assert param("epoch") == M32 - STRIDE + 1, param("epoch")  # the scrub ends on 0
    after = (b * STRIDE + 1) % M32
    for k, v in enumerate(variants):
        fam(v, 100 + k)
        expect_epoch(after + (k + 1) * STRIDE, "after %s" % X.family)
        done += 1
    lib.b200mpi_set_max_blocks(0)
    mpi.Barrier()
    return {"checked": done, "epoch": param("epoch")}


def scenario_wrap_hostpipe(a):
    """A pipelined host-slice Allreduce (64 KiB chunks, one launch each) whose six chunks straddle the
    scrub that ends on 0: three before it, three after.  --variants "dtype:pageable|pinned:count:in|out"."""
    lib = L.load()
    rank, n = mpi.Rank(), mpi.Size()
    for k, v in (("pipe_min_bytes", 65536), ("pipe_chunk_bytes", 65536), ("bounce_chunk_bytes", 65536)):
        if lib.b200mpi_set_param(k.encode(), v):
            raise RuntimeError(L.last_error())
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS["twoshot"])
    dn, mem, count, inplace = parse_variants(X.variants)[0]
    dt = W.DTYPES[dn]
    if -(-count * np.dtype(dt).itemsize // 65536) != 6:
        raise AssertionError("the message must make six chunks")
    ins = W.inputs_for(dt, n, count, salt=count % 83)
    want = O.allreduce(ins)
    frees = []
    if mem == "pageable":
        send, recv = np.array(ins[rank]), np.zeros(count, dtype=dt)
    else:
        send, p = W.pinned_array(count, dt)
        recv, q = W.pinned_array(count, dt)
        frees += [p, q]
        send[:] = ins[rank]
    place((M32 - 4 * STRIDE + 1) % M32)
    e0 = next_start()
    mpi.Allreduce(send, send if inplace else recv)
    check_equal(send if inplace else recv, want, "hostpipe %s %s inplace=%s across the wrap" % (dn, mem, inplace))
    if not inplace:
        check_equal(send, ins[rank], "hostpipe: send untouched")
    moved = (param("epoch") - e0) % M32 // STRIDE
    if moved != 6 + 1:
        raise AssertionError("hostpipe %s: %d strides, expected six chunks and the scrub" % (dn, moved))
    for p in frees:
        lib.b200mpi_host_free(p)
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
    mpi.Barrier()
    return {"checked": 1}


def scenario_wrap_mismatch(a):
    """A mismatched call is the last launch before the scrub that ends on 0 (--family count: ranks
    disagree on the count; --family alltoallv: one rank's recv table is off by one).  Every rank gets
    B200MPI_ERR_PEER with no buffer touched; the resync steps over the scrub's index, so the epoch
    crosses 0 without a launch, and the next call (start 1) is correct."""
    lib = L.load()
    rank, n = mpi.Rank(), mpi.Size()
    m = [[3 + 5 * i + 2 * j for j in range(n)] for i in range(n)]
    srow, rcol = A.row(m, rank), A.col(m, rank)
    st = lambda t: (ctypes.c_size_t * n)(*t)  # noqa: E731
    x0, y0 = gfill(np.float32, SEED + rank, 1000), sentinel(np.float32, 1000)
    x, y = make_buffer("heap", x0), make_buffer("heap", y0)
    place((M32 - 2 * STRIDE + 1) % M32)
    if X.family == "count":
        rc = lib.b200mpi_allreduce(x.ptr, y.ptr, 1000 if rank == 0 else 999, L.F32, L.SUM, L.DEVICE)
    else:
        off = list(rcol)
        off[0] += 1
        rc = lib.b200mpi_alltoallv(x.ptr, st(srow), y.ptr, st(off if rank == 1 else rcol), L.F32, L.DEVICE)
    assert rc == L.ERR_PEER, (rc, L.last_error())
    check_equal(y.to_host(), y0, "%s mismatch before the wrap: recv untouched" % X.family)
    check_equal(x.to_host(), x0, "%s mismatch before the wrap: send untouched" % X.family)
    expect_epoch(1, "after the mismatch and its resync across 0")
    if X.family == "count":
        ins = [gfill(np.float32, SEED + r, 1000) for r in range(n)]
        mpi.Allreduce(x, y)
        check_equal(y.to_host(), O.allreduce(ins, order=O.ORDER_TREE if n in (2, 4, 8) else O.ORDER_RANK), "allreduce after the mismatch")
    else:
        sends = [gfill(np.float32, SEED + 11 + i, sum(m[i])) for i in range(n)]
        send = make_buffer("heap", sends[rank])
        got, _ = mpi.Alltoallv(send, srow, y[:sum(rcol)], rcol)
        check_equal(read_buffer(got), A.alltoallv(sends, m, rank), "alltoallv after the mismatch")
        free_buffer(send)
    expect_epoch(1 + STRIDE, "after the first call past the wrap")
    x.free()
    y.free()
    mpi.Barrier()
    return {"checked": 2}


def epoch_after(e, k):
    """The epoch after k launches through next_comm from epoch e (a due scrub takes one stride more)."""
    for _ in range(k):
        if scrub_due(e):
            e = (e + STRIDE) % M32
        e = (e + STRIDE) % M32
    return e


def ll_call(kind, count, salt, what, clears=False):
    """One LL Allreduce, checked bit for bit.  An LL kernel takes no epoch; the lane clearing at the
    wrap runs two barriers, one stride each, so the epoch shows whether the lanes were cleared."""
    e0 = param("epoch")
    ll_call_unchecked(kind, count, salt, what)
    want = epoch_after(e0, 2) if clears else e0
    if param("epoch") != want:
        raise AssertionError("LL %s: epoch %d -> %d, expected %d (%s)" % (what, e0, param("epoch"), want,
                                                                       "lanes cleared once" if clears else "no clearing"))


def ll_call_unchecked(kind, count, salt, what):
    rank, n = mpi.Rank(), mpi.Size()
    ins = W.inputs_for(np.float32, n, count, salt=salt)
    send = make_buffer(kind, ins[rank])
    recv = make_buffer(kind, np.zeros(count, dtype=np.float32))
    mpi.Allreduce(send, recv, mpi.SUM)
    check_equal(read_buffer(recv), O.allreduce(ins, order=O.ORDER_RANK), "LL %s %s count=%d" % (what, kind, count))
    free_buffer(send)
    free_buffer(recv)


def scenario_ll_wrap(a):
    """LL Allreduce at the sequence wrap (start B200MPI_LL_SEQ_START = 2^32 - 5).

    plain:  four 1-element calls, then the call that would get sequence 0 is the first one larger than
            any before it (40,000 f32): its lanes beyond one cell still hold the zeros of Init, which
            match sequence 0.  Rank 1 sleeps before it, so rank 0's kernel reads before any peer cell
            lands.  Then 40,000 and smaller calls alternate.
    resync: a 40,000-element call shortly before the wrap, then a mismatched non-LL call whose resync
            moves the sequence from 2^32 - 2 across 0; the calls after it must be exact."""
    lib = L.load()
    rank = mpi.Rank()
    kind = a.kinds
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS["ll"])
    done = 0
    start = param("ll_seq")
    assert start == M32 - 5, start
    if X.family == "plain":
        for k in range(4):
            ll_call(kind, 1, k, "before the wrap")
        assert param("ll_seq") == M32 - 1, param("ll_seq")
        if rank == 1:
            time.sleep(1.0)
        ll_call(kind, 40000, 50, "the wrap call", clears=True)
        done += 5
    else:
        ll_call(kind, 40000, 60, "large, before the wrap")  # 2^32 - 4
        ll_call(kind, 3, 61, "small, before the wrap")      # 2^32 - 3
        ll_call(kind, 3, 62, "small, before the wrap")      # 2^32 - 2
        assert param("ll_seq") == M32 - 2, param("ll_seq")
        x = mpi.Alloc(1000, np.float32)
        lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS["twoshot"])
        rc = lib.b200mpi_allreduce(x.ptr, x.ptr, 1000 if rank == 0 else 999, L.F32, L.SUM, L.DEVICE)
        assert rc == L.ERR_PEER, (rc, L.last_error())
        x.free()
        lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS["ll"])
        if rank == 1:
            time.sleep(1.0)
        ll_call(kind, 40000, 63, "the first call after a resync across the wrap", clears=True)
        done += 4
    seq = param("ll_seq")
    if not (0 < seq < 16):
        raise AssertionError("the sequence did not restart: ll_seq %d" % seq)
    for k in range(6):
        ll_call(kind, 40000 if k % 2 == 0 else 1 + 997 * k, 70 + k, "after the wrap")
        done += 1
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
    mpi.Barrier()
    return {"checked": done, "ll_seq": param("ll_seq")}


X = None  # this world's --family / --variants / --boundary / --max-blocks (set in __main__)
def scenario_across(a):
    """One of _worker.py's scenarios (--family), then the epoch and LL sequence it ended on, so that
    the test can check that the run crossed the boundary it was started below."""
    out = W.SCENARIOS[X.family](a)
    out.update({"epoch": param("epoch"), "ll_seq": param("ll_seq")})
    return out


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_")})

if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--family", default="")
    ap.add_argument("--variants", default="")
    ap.add_argument("--boundary", default=str(1 << 20))
    ap.add_argument("--max-blocks", dest="max_blocks", default="")
    X, rest = ap.parse_known_args()
    sys.argv = [sys.argv[0]] + rest  # _worker.main parses the rest
    W.main()
