"""numpy model of the passive-target calls (b200mpi_get_accumulate, _fetch_and_op, _compare_and_swap,
_win_lock / _win_unlock).

It extends _rma_ref's element rules (combine, ftz32) with REPLACE (target = origin) and NO_OP (target
unchanged), the fetch (every call returns the target's previous bits, exactly, whatever the op does to
the target), compare-and-swap, and a sequential model of lock-protected read-modify-write rounds: a
lock makes each round's Get, update and Put one indivisible step, so any serial order of the rounds
gives the final records."""
import numpy as np

from _rma_ref import MAX, MIN, SUM, combine, ftz32  # noqa: F401

REPLACE, NO_OP = 3, 4
OPS = {"sum": SUM, "max": MAX, "min": MIN, "replace": REPLACE, "no_op": NO_OP}


def apply(a, b, op):
    """The target's new values: a op b, with the one-sided ops."""
    a = np.asarray(a)
    if op == REPLACE:
        return np.array(b, dtype=a.dtype, copy=True)
    if op == NO_OP:
        return a.copy()
    return combine(a, np.asarray(b, dtype=a.dtype), op)


def fetch_op(target, origin, op):
    """Get_accumulate / Fetch_and_op on target values: -> (fetched, new target).  The fetch is the
    previous bits exactly, never flushed or canonicalised."""
    target = np.asarray(target)
    return target.copy(), apply(target, origin, op)


def compare_and_swap(target, origin, compare):
    """-> (fetched, new target): origin is stored where the old value equals compare."""
    target = np.asarray(target, dtype=np.int64)
    return target.copy(), np.where(target == compare, np.int64(origin), target).astype(np.int64)


def serial(init, calls):
    """Fetching calls (op, origin) on one element, applied in the given order: -> (fetched values in
    call order, final value).  Concurrent atomics produce the result of some such order."""
    cur = np.asarray([init])
    fetched = []
    for op, origin in calls:
        old, cur = fetch_op(cur, [origin], op)
        fetched.append(old[0])
    return fetched, cur[0]


def locked_rounds(n, rounds, length, visits):
    """Each of n ranks runs `rounds` rounds; in each it visits the targets visits(rank, round) and, under
    an exclusive lock on each, Gets the target's record of `length` int64, adds 1 to every element and
    Puts it back.  -> every target's final record.  Rank-major order is one serial order of the rounds."""
    recs = [np.zeros(length, dtype=np.int64) for _ in range(n)]
    for rank in range(n):
        for r in range(rounds):
            for t in visits(rank, r):
                recs[t] = recs[t] + 1
    return recs


def same_bits(a, b, nan_equal=False):
    """Byte-for-byte equality; nan_equal: any two NaNs match (an arithmetic NaN result's payload is the
    hardware's choice, so a SUM into a NaN is compared that way)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    eq = a.view(np.uint8).reshape(a.size, -1) == b.view(np.uint8).reshape(b.size, -1)
    ok = eq.all(axis=1) if a.size else np.ones(0, bool)
    if nan_equal and a.dtype.kind == "f":
        ok = ok | (np.isnan(a) & np.isnan(b))
    return bool(ok.all())
