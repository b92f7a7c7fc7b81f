"""One rank of a test world for generalized active-target synchronisation (Post, Start, Complete, Wait,
Test).  Usage as _worker.py: _pscw_worker.py <scenario> --out FILE [scenario args] -mpi-* flags.
Windows are guarded views (_rma_atomic_worker.Wnd) whose bodies and guards are checked byte for byte
against their model after each epoch that wrote them."""
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _worker as W  # noqa: E402
from _rma_atomic_worker import Wnd  # noqa: E402
from _worker import L, mpi  # noqa: E402


def ring(rank, n):
    """(left, right, the distinct neighbours in order)."""
    left, right = (rank - 1) % n, (rank + 1) % n
    return left, right, sorted({left, right})


def expect_code(call, code, what):
    try:
        call()
    except mpi.MpiError as e:
        assert e.code == code, (what, e.code, code, str(e))
        return
    raise AssertionError("%s succeeded (wanted error %d)" % (what, code))


def with_watchdog_ms(ms, call):
    """call() with the watchdog_ms knob at `ms`, restored afterwards (no collective runs meanwhile)."""
    old = L.get_param("watchdog_ms")
    assert L.load().b200mpi_set_param(b"watchdog_ms", ms) == 0
    try:
        return call()
    finally:
        assert L.load().b200mpi_set_param(b"watchdog_ms", old) == 0


def scenario_pscw_halo(a):
    """A ring halo exchange, one PSCW epoch per iteration with values that change every iteration.
    Window: [ghost left G | interior I | ghost right G] int64.  The target writes its interior, then
    posts to its neighbours; after Start each rank Gets both neighbours' interiors (the values they
    held at their post) and Puts its first G interior elements into the left neighbour's right ghost
    cells and its last G into the right neighbour's left ghost cells; after Complete and Wait the
    target's window is checked exactly, guards included."""
    rank, n = mpi.Rank(), mpi.Size()
    G, I_ = 3, 29
    iters = 200
    left, right, nbrs = ring(rank, n)

    def interior(r, it):
        return (np.arange(I_, dtype=np.int64) * 7919 + r * 1000003 + it * 65537) ^ (it << 40)

    w = Wnd(np.int64, 2 * G + I_, 8, 101, lambda r: np.zeros(2 * G + I_, dtype=np.int64))
    for it in range(iters):
        mine = interior(rank, it)
        w.buf.view[G:G + I_].copy_from_host(mine)
        w.win.Post(nbrs)
        w.win.Start(nbrs)
        for r in nbrs:
            got = w.win.Get(np.empty(I_, dtype=np.int64), r, G)
            assert np.array_equal(got, interior(r, it)), ("Get after Start", it, r)
        w.win.Put(mine[:G], left, G + I_)
        w.win.Put(mine[-G:], right, 0)
        w.win.Complete()
        w.win.Wait()
        body = np.concatenate([interior(left, it)[-G:], mine, interior(right, it)[:G]])
        w.images[rank] = body.view(np.uint8).copy()
        w.check("halo iteration %d" % it)
    mpi.Barrier()
    w.free()
    mpi.Barrier()
    return {"checked": iters}


def scenario_pscw_star(a):
    """Rank 0 posts to every rank; every rank starts on {0} and Accumulates int64 SUM into rank 0's
    window; after Wait rank 0's window is the exact (wrapping) numpy sum.  Five epochs, values near
    the int64 limits."""
    rank, n = mpi.Rank(), mpi.Size()
    E = 17
    i64 = np.iinfo(np.int64)
    w = Wnd(np.int64, E, 16, 111, lambda r: np.zeros(E, dtype=np.int64))
    total = np.zeros(E, dtype=np.int64)

    def contrib(r, ep):
        v = np.arange(E, dtype=np.int64) * (r + 1) * (ep + 3) - r
        v[0] = i64.max - r if ep % 2 else i64.min + r
        return v

    for ep in range(5):
        if rank == 0:
            w.win.Post(range(n))
        w.win.Start([0])
        w.win.Accumulate(contrib(rank, ep), 0, 0, op=mpi.SUM)
        w.win.Complete()
        with np.errstate(over="ignore"):
            for r in range(n):
                total = total + contrib(r, ep)
        if rank == 0:
            w.win.Wait()
            w.images[0] = total.view(np.uint8).copy()
            w.check("star epoch %d" % ep)
    mpi.Barrier()
    w.check("star, every rank")
    w.free()
    mpi.Barrier()
    return {"checked": 5}


def scenario_pscw_disjoint(a):
    """n = 4: the pairs (0, 1) and (2, 3) run 10 and 300 epochs on one window with no collective
    between; each rank Puts an epoch-stamped record into its partner's window, and each target checks
    its window after every Wait.  Only the final Barrier joins the pairs."""
    rank, n = mpi.Rank(), mpi.Size()
    assert n == 4
    E = 8
    partner = rank ^ 1
    epochs = 10 if rank < 2 else 300

    def rec(r, ep):
        return np.arange(E, dtype=np.int64) + r * 100000 + ep * 1000

    w = Wnd(np.int64, E, 0, 121, lambda r: np.zeros(E, dtype=np.int64))
    for ep in range(epochs):
        w.win.Post([partner])
        w.win.Start([partner])
        w.win.Put(rec(rank, ep), partner, 0)
        w.win.Complete()
        w.win.Wait()
        w.images[rank] = rec(partner, ep).view(np.uint8).copy()
        w.check("pair epoch %d" % ep)
    mpi.Barrier()
    w.check("after the pairs joined")
    w.free()
    mpi.Barrier()
    return {"checked": epochs}


def scenario_pscw_counts(a):
    """Post and Complete are one launch each, Start and Wait one launch each when their peers are
    already there, Test one launch; an empty group launches nothing.  No call takes an epoch or uses
    heap."""
    lib, rank, n = L.load(), mpi.Rank(), mpi.Size()
    left, right, _ = ring(rank, n)
    w = Wnd(np.int64, 8, 0, 131, lambda r: np.zeros(8, dtype=np.int64))
    used = ctypes.c_size_t()

    def measured(name, call, launches):
        assert lib.b200mpi_heap_info(None, ctypes.byref(used), None) == 0
        used0, epoch0, l0 = used.value, L.get_param("epoch"), lib.b200mpi_launch_count()
        r = call()
        assert lib.b200mpi_launch_count() - l0 == launches, (name, lib.b200mpi_launch_count() - l0, launches)
        assert L.get_param("epoch") == epoch0, (name, "took an epoch")
        assert lib.b200mpi_heap_info(None, ctypes.byref(used), None) == 0 and used.value == used0, (name, "used heap")
        return r

    measured("post", lambda: w.win.Post([left]), 1)
    mpi.Barrier()                                          # every target has posted
    measured("start", lambda: w.win.Start([right]), 1)
    measured("complete", lambda: w.win.Complete(), 1)
    mpi.Barrier()                                          # every origin has completed
    measured("wait", lambda: w.win.Wait(), 1)
    measured("post again", lambda: w.win.Post([left]), 1)
    mpi.Barrier()
    measured("start again", lambda: w.win.Start([right]), 1)
    measured("complete again", lambda: w.win.Complete(), 1)
    mpi.Barrier()
    assert measured("test", lambda: w.win.Test(), 1) is True
    for name, call in (("empty post", lambda: w.win.Post([])), ("empty start", lambda: w.win.Start(())),
                       ("empty complete", lambda: w.win.Complete()), ("empty wait", lambda: w.win.Wait()),
                       ("empty post 2", lambda: w.win.Post(np.array([], dtype=np.int64)))):
        measured(name, call, 0)
    assert measured("empty test", lambda: w.win.Test(), 0) is True
    mpi.Barrier()
    w.check("counts: nothing written")
    w.free()
    mpi.Barrier()
    return {"checked": 13}


def scenario_pscw_self(a):
    """A group containing this rank.  World of one: group {0} for 65,540 epochs, so the 16-bit
    counters wrap, with a Put into the own window checked every 4,096 epochs and at the end.  Larger
    worlds: Post to {self, left} and Start on {self, right}, Put into both, checked after Wait."""
    rank, n = mpi.Rank(), mpi.Size()
    w = Wnd(np.int64, 4, 8, 141, lambda r: np.zeros(4, dtype=np.int64))
    if n == 1:
        epochs = 65540
        lib, wid = L.load(), w.win.id
        grp = (ctypes.c_int * 1)(0)
        for ep in range(epochs):
            check = ep % 4096 == 0 or ep == epochs - 1
            assert lib.b200mpi_win_post(grp, 1, wid) == 0, (ep, L.last_error())
            assert lib.b200mpi_win_start(grp, 1, wid) == 0, (ep, L.last_error())
            if check:
                v = np.array([ep, -ep, ep * 3, 7], dtype=np.int64)
                w.win.Put(v, 0, 0)
            assert lib.b200mpi_win_complete(wid) == 0, (ep, L.last_error())
            assert lib.b200mpi_win_wait(wid) == 0, (ep, L.last_error())
            if check:
                w.images[0] = v.view(np.uint8).copy()
                w.check("self epoch %d" % ep)
        w.free()
        return {"checked": epochs}
    left, right, _ = ring(rank, n)
    for ep in range(20):
        w.win.Post([rank, left])
        w.win.Start([right, rank])
        w.win.Put(np.array([rank, ep], dtype=np.int64), rank, 0)
        w.win.Put(np.array([rank, ep], dtype=np.int64), right, 2)
        w.win.Complete()
        w.win.Wait()
        w.images[rank] = np.array([rank, ep, left, ep], dtype=np.int64).view(np.uint8).copy()
        w.check("self and neighbour, epoch %d" % ep)
    mpi.Barrier()
    w.free()
    mpi.Barrier()
    return {"checked": 20}


def scenario_pscw_errors(a):
    """Every argument and state error returns ERR_ARG and launches nothing; the window and the epochs
    are unchanged (an epoch that was open still closes normally)."""
    lib, rank, n = L.load(), mpi.Rank(), mpi.Size()
    left, right, nbrs = ring(rank, n)
    w = Wnd(np.float64, 16, 8, 151, lambda r: np.arange(16, dtype=np.float64) + 100 * r)
    gone = mpi.WinCreate(None)
    gone.Free()
    wid = w.win.id

    def grp(*ranks):
        return (ctypes.c_int * max(len(ranks), 1))(*ranks)

    flag = ctypes.c_int(7)
    ok1 = grp(right)
    cases = [
        ("post unknown window", lambda: lib.b200mpi_win_post(ok1, 1, wid + 100)),
        ("start unknown window", lambda: lib.b200mpi_win_start(ok1, 1, wid + 100)),
        ("complete unknown window", lambda: lib.b200mpi_win_complete(-1)),
        ("wait unknown window", lambda: lib.b200mpi_win_wait(wid + 100)),
        ("test unknown window", lambda: lib.b200mpi_win_test(wid + 100, ctypes.byref(flag))),
        ("post freed window", lambda: lib.b200mpi_win_post(ok1, 1, gone.id)),
        ("start freed window", lambda: lib.b200mpi_win_start(ok1, 1, gone.id)),
        ("complete freed window", lambda: lib.b200mpi_win_complete(gone.id)),
        ("wait freed window", lambda: lib.b200mpi_win_wait(gone.id)),
        ("test freed window", lambda: lib.b200mpi_win_test(gone.id, ctypes.byref(flag))),
    ]
    for name, call in (("post", lib.b200mpi_win_post), ("start", lib.b200mpi_win_start)):
        cases += [
            (name + " NULL group", lambda call=call: call(None, 1, wid)),
            (name + " negative count", lambda call=call: call(ok1, -1, wid)),
            (name + " count > size", lambda call=call: call(grp(*range(n), 0), n + 1, wid)),
            (name + " rank = size", lambda call=call: call(grp(n), 1, wid)),
            (name + " rank -1", lambda call=call: call(grp(-1), 1, wid)),
            (name + " duplicate", lambda call=call: call(grp(right, right), 2, wid)),
        ]
    cases += [
        ("complete without start", lambda: lib.b200mpi_win_complete(wid)),
        ("wait without post", lambda: lib.b200mpi_win_wait(wid)),
        ("test without post", lambda: lib.b200mpi_win_test(wid, ctypes.byref(flag))),
    ]
    l0 = lib.b200mpi_launch_count()
    done = 0
    for name, call in cases:
        rc = call()
        assert rc == L.ERR_ARG, (name, rc, L.last_error())
        done += 1
    assert flag.value == 7, "a refused test wrote its flag"
    assert lib.b200mpi_launch_count() == l0, "a refused call launched"
    # open epochs: a second post / start is refused, then they close normally
    w.win.Post(nbrs)
    mpi.Barrier()
    w.win.Start(nbrs)
    l1 = lib.b200mpi_launch_count()
    for name, call in (("post while exposed", lambda: lib.b200mpi_win_post(grp(left), 1, wid)),
                       ("empty post while exposed", lambda: lib.b200mpi_win_post(None, 0, wid)),
                       ("start while accessing", lambda: lib.b200mpi_win_start(grp(right), 1, wid)),
                       ("empty start while accessing", lambda: lib.b200mpi_win_start(None, 0, wid)),
                       ("test NULL flag", lambda: lib.b200mpi_win_test(wid, None))):
        rc = call()
        assert rc == L.ERR_ARG, (name, rc, L.last_error())
        done += 1
    assert lib.b200mpi_launch_count() == l1, "a refused call launched"
    w.win.Complete()
    w.win.Wait()
    mpi.Barrier()
    w.check("errors: nothing written")
    w.free()
    mpi.Barrier()
    return {"checked": done}


def scenario_pscw_timeout(a):
    """watchdog_ms = 2000.  Rank 1's Start before rank 0 has posted times out in about 2 s and leaves
    no access epoch; after rank 0's late Post the Start succeeds.  Then rank 0's Wait for rank 1,
    which has started but not completed, times out and stays open: Test is False; after rank 1's late
    Complete, Wait succeeds and rank 1's Put is there."""
    rank = mpi.Rank()
    lib = L.load()
    w = Wnd(np.int64, 4, 0, 161, lambda r: np.zeros(4, dtype=np.int64))
    mpi.Barrier()
    if rank == 1:
        t0 = time.time()
        with_watchdog_ms(2000, lambda: expect_code(lambda: w.win.Start([0]), L.ERR_TIMEOUT, "start without a post"))
        dt = time.time() - t0
        assert 1.9 < dt < 60, dt
        assert lib.b200mpi_win_complete(w.win.id) == L.ERR_ARG, "the timed-out start left an access epoch open"
    mpi.Barrier()
    if rank == 0:
        w.win.Post([1])
    mpi.Barrier()
    if rank == 1:
        w.win.Start([0])                                   # the late post is seen
    mpi.Barrier()
    if rank == 0:
        t0 = time.time()
        with_watchdog_ms(2000, lambda: expect_code(lambda: w.win.Wait(), L.ERR_TIMEOUT, "wait before the complete"))
        dt = time.time() - t0
        assert 1.9 < dt < 60, dt
        assert w.win.Test() is False
        expect_code(lambda: w.win.Post([1]), L.ERR_ARG, "the exposure epoch stayed open")
    mpi.Barrier()
    if rank == 1:
        w.win.Put(np.array([11, 22, 33, 44], dtype=np.int64), 0, 0)
        w.win.Complete()
    mpi.Barrier()
    if rank == 0:
        w.win.Wait()
        w.images[0] = np.array([11, 22, 33, 44], dtype=np.int64).view(np.uint8).copy()
    w.check("timeout")
    w.win.Fence()
    w.free()
    mpi.Barrier()
    return {"checked": 4}


def scenario_pscw_partial(a):
    """n = 3, watchdog_ms = 2000: rank 0's Start on {1, 2}, when only rank 1 has posted, times out and
    opens no epoch; rank 1's post is not consumed, so after rank 2's late Post the next Start on
    {1, 2} succeeds, and rank 0's Puts reach both targets by their Wait."""
    lib, rank, n = L.load(), mpi.Rank(), mpi.Size()
    assert n == 3
    w = Wnd(np.int64, 2, 0, 165, lambda r: np.zeros(2, dtype=np.int64))
    if rank == 1:
        w.win.Post([0])
    mpi.Barrier()
    if rank == 0:
        t0 = time.time()
        with_watchdog_ms(2000, lambda: expect_code(lambda: w.win.Start([1, 2]), L.ERR_TIMEOUT, "start with one target missing"))
        dt = time.time() - t0
        assert 1.9 < dt < 60, dt
        assert lib.b200mpi_win_complete(w.win.id) == L.ERR_ARG, "the timed-out start left an access epoch open"
    mpi.Barrier()
    if rank == 2:
        w.win.Post([0])
    mpi.Barrier()
    if rank == 0:
        l0 = lib.b200mpi_launch_count()
        w.win.Start([1, 2])                                # rank 1's earlier post still counts
        assert lib.b200mpi_launch_count() - l0 == 1, "both posts were there: one poll launch"
        for t in (1, 2):
            w.win.Put(np.array([t * 10, t * 10 + 1], dtype=np.int64), t, 0)
        w.win.Complete()
    else:
        w.win.Wait()
        w.images[rank] = np.array([rank * 10, rank * 10 + 1], dtype=np.int64).view(np.uint8).copy()
    w.check("partial arrival")
    mpi.Barrier()
    w.free()
    mpi.Barrier()
    return {"checked": 3}


def scenario_pscw_fence(a):
    """Fence and Free by a rank with an open exposure or access epoch: ERR_ARG there, ERR_PEER on every
    other rank (a world of one: ERR_ARG, nothing launched); the window stays live and the epoch open.
    Once the epochs close the next fence works; then fence epochs and PSCW epochs alternate on one
    window."""
    lib, rank, n = L.load(), mpi.Rank(), mpi.Size()
    E = 2 * n
    w = Wnd(np.int64, E, 8, 171, lambda r: np.zeros(E, dtype=np.int64))
    h = n - 1

    def refused(holders, what="fence"):
        l0 = lib.b200mpi_launch_count()
        rc = lib.b200mpi_win_fence(w.win.id) if what == "fence" else lib.b200mpi_win_free(w.win.id)
        want = L.ERR_ARG if rank in holders else L.ERR_PEER
        assert rc == want, (what, holders, rc, want, L.last_error())
        if n == 1:
            assert lib.b200mpi_launch_count() == l0, "a world of one launched a fence"

    if rank == h:
        w.win.Post([0])                                    # h: exposure open
        w.win.Lock(h, mpi.LOCK_SHARED)                     # and a lock held on the same window
    refused({h})
    if rank == h:                                          # the refusal names both, then the epoch alone
        msg = L.last_error()
        assert "lock" in msg and "epoch" in msg, msg
        w.win.Unlock(h)
    refused({h})
    if rank == h:
        msg = L.last_error()
        assert "epoch" in msg and "lock" not in msg, msg
    refused({h}, "free")
    if rank == 0:
        w.win.Start([h])                                   # 0: access open too
    refused({0, h})
    if rank == 0:
        w.win.Put(np.array([5, 6], dtype=np.int64), h, 0)
        w.win.Complete()
    refused({h}, "free")
    if rank == h:
        w.win.Wait()
    w.win.Fence()
    body = np.zeros(E, dtype=np.int64)
    if rank == h:
        body[:2] = [5, 6]
    w.images[rank] = body.view(np.uint8).copy()
    w.check("after the epochs closed")
    left, right, nbrs = ring(rank, n)
    for rnd in range(4):
        # a fence epoch: every rank Puts into its right neighbour's slot `rank`.  The opening fence
        # also ends every rank's check of its window (after the epochs closed, or after the last
        # PSCW round) before any rank writes into it again.
        w.win.Fence()
        w.win.Put(np.array([rnd, rank], dtype=np.int64), right, 2 * rank if n > 1 else 0)
        w.win.Fence()
        body[2 * left:2 * left + 2] = [rnd, left]
        w.images[rank] = body.view(np.uint8).copy()
        w.check("fence round %d" % rnd)
        w.win.Fence()                                      # the target's local read ends before the next writes
        # a PSCW epoch on the same window: the same exchange, values negated
        w.win.Post(nbrs)
        w.win.Start(nbrs)
        w.win.Put(np.array([-rnd - 1, -rank], dtype=np.int64), right, 2 * rank if n > 1 else 0)
        w.win.Complete()
        w.win.Wait()
        body[2 * left:2 * left + 2] = [-rnd - 1, -left]
        w.images[rank] = body.view(np.uint8).copy()
        w.check("pscw round %d" % rnd)
    mpi.Barrier()
    w.free()
    mpi.Barrier()
    return {"checked": 8}


def scenario_pscw_cells(a):
    """One window stays in a PSCW epoch (exposure and access open) while a few hundred others are
    created and freed, each reusing the same cell.  On each new window a Start before any Post times
    out (its posted counters are clear) and a Test right after Post is False (its completed counters
    are clear); then one epoch's Put arrives."""
    rank, n = mpi.Rank(), mpi.Size()
    left, right, _ = ring(rank, n)
    keep = Wnd(np.int64, 4, 0, 181, lambda r: np.zeros(4, dtype=np.int64))
    keep.win.Post([left])
    mpi.Barrier()
    keep.win.Start([right])
    mem = mpi.Alloc(4, np.int64).copy_from_host(np.zeros(4, dtype=np.int64))
    cycles = (300 if n == 1 else 150)
    for i in range(cycles):
        w = mpi.WinCreate(mem)
        assert w.id > keep.win.id
        with_watchdog_ms(1, lambda: expect_code(lambda: w.Start([right]), L.ERR_TIMEOUT, "start on a new window before any post"))
        mpi.Barrier()
        w.Post([left])
        assert w.Test() is False, ("stale completed counter", i)
        mpi.Barrier()
        w.Start([right])
        w.Put(np.array([i, rank], dtype=np.int64), right, 0)
        w.Complete()
        w.Wait()
        assert mem.to_host()[:2].tolist() == [i, left], (i, mem.to_host())
        w.Free()
    keep.win.Complete()
    keep.win.Wait()
    keep.win.Fence()
    mem.free()
    keep.free()
    mpi.Barrier()
    return {"checked": cycles}


def scenario_pscw_control_only(a):
    """Control plane only: all five entries refuse with B200MPI_ERR_NO_DEVICE, through the C ABI and the facade."""
    lib = L.load()
    grp = (ctypes.c_int * 1)(0)
    flag = ctypes.c_int(5)
    assert lib.b200mpi_win_post(grp, 1, 0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_win_start(grp, 1, 0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_win_complete(0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_win_wait(0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_win_test(0, ctypes.byref(flag)) == L.ERR_NO_DEVICE and flag.value == 5
    w = mpi.Win(0)
    for call in (lambda: w.Post([0]), lambda: w.Start([0]), lambda: w.Complete(), lambda: w.Wait(), lambda: w.Test()):
        expect_code(call, L.ERR_NO_DEVICE, "data call without a device")
    return {"checked": 10}


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_pscw_")})

if __name__ == "__main__":
    W.main()
