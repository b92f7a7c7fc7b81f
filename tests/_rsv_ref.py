"""ReduceScatterv restated for the tests (test infrastructure only): rank j receives the rank-order
reduction of block j of every rank's send, where block j is counts[j] elements at displacement
counts[0] + ... + counts[j-1].

rsv_oracle takes that from the C oracle (oracle_allreduce in ORDER_RANK over the whole sends, sliced
at the displacements); rsv_np restates it in numpy with the kernels' operators, and the CPU tests pin
the two against each other, against hand-worked values and, on uniform tables, against
oracle_reduce_scatter."""
import numpy as np

from _scan_ref import apply
from oracle import oracle as O


def displs(counts):
    """[counts[0] + ... + counts[j-1] for j = 0..n]: the block boundaries, total last."""
    return [int(x) for x in np.concatenate([[0], np.cumsum(np.asarray(counts, dtype=np.int64))])]


def rsv_np(sends, counts, op):
    """Every rank's result, in rank order."""
    d = displs(counts)
    xs = [np.ascontiguousarray(s).reshape(-1) for s in sends]
    out = []
    for j in range(len(counts)):
        acc = xs[0][d[j]:d[j + 1]].copy()
        for x in xs[1:]:
            acc = apply(op, acc, x[d[j]:d[j + 1]])
        out.append(acc)
    return out


def rsv_oracle(sends, counts, op, rank):
    """What `rank` receives: oracle_allreduce of the whole sends in rank order, sliced at its block."""
    d = displs(counts)
    if d[-1] == 0:
        return np.zeros(0, dtype=np.asarray(sends[0]).dtype)
    return O.allreduce(sends, op=op, order=O.ORDER_RANK)[d[rank]:d[rank + 1]]


def balanced(total, n):
    """The balanced split of `total` elements: the first total % n ranks hold one more."""
    return [total // n + (1 if r < total % n else 0) for r in range(n)]


def skewed(total, n, heavy=None):
    """One rank (the last by default) holds most of `total`; every other rank a few elements, some 0."""
    heavy = n - 1 if heavy is None else heavy
    small = [0 if r % 3 == 1 else 3 + 5 * r for r in range(n)]
    small[heavy] = 0
    small[heavy] = max(total - sum(small), 0)
    return small
