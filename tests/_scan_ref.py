"""Scan and Exscan restated for the tests (test infrastructure only): what rank r receives is the
rank-order reduction of ranks 0..r (Scan) or 0..r-1 (Exscan; rank 0 receives nothing).

scan_oracle takes that reduction from the C oracle (oracle_allreduce in ORDER_RANK over a prefix of
the inputs); scan_np restates it in numpy with the kernels' operators, and the CPU tests pin the two
against each other and against hand-worked values."""
import numpy as np

from oracle import oracle as O


def apply(op, a, b):
    """Op::apply of kernels.cuh: a + b (i64 wraps), b > a ? b : a, b < a ? b : a."""
    with np.errstate(over="ignore", invalid="ignore"):
        if op == O.SUM:
            if a.dtype == np.int64:
                return (a.view(np.uint64) + b.view(np.uint64)).view(np.int64)
            return a + b
        if op == O.MAX:
            return np.where(b > a, b, a)
        return np.where(b < a, b, a)


def scan_np(inputs, op, exclusive=False):
    """Every rank's result, in rank order; None for rank 0 of an Exscan."""
    out, acc = [], None
    for x in inputs:
        x = np.ascontiguousarray(x).reshape(-1)
        if exclusive:
            out.append(None if acc is None else acc.copy())
        acc = x.copy() if acc is None else apply(op, acc, x)
        if not exclusive:
            out.append(acc.copy())
    return out


def scan_oracle(inputs, op, rank, exclusive=False):
    """What `rank` receives, from oracle_allreduce over the prefix of ranks; None for rank 0 of an Exscan."""
    k = rank if exclusive else rank + 1
    if k == 0:
        return None
    return O.allreduce(inputs[:k], op=op, order=O.ORDER_RANK)
