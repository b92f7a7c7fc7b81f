"""Restatement of Alltoallv in numpy -- TEST INFRASTRUCTURE.

The exchange is a pure permutation of elements, so the restatement is exact for every dtype.  A
matrix m of block sizes describes a whole call: m[i][j] is the number of elements rank i sends to
rank j, so rank i passes send_counts = m[i] and recv_counts = [m[k][i] for k]."""
import numpy as np


def row(m, i):
    return [int(c) for c in m[i]]


def col(m, i):
    return [int(m[k][i]) for k in range(len(m))]


def alltoallv(sends, m, me):
    """sends[i] is rank i's send buffer (sum(m[i]) elements, block j for rank j packed in rank
    order); returns rank me's recv: the blocks from ranks 0..n-1 for me, packed in rank order."""
    n = len(m)
    parts = []
    for k in range(n):
        src = np.asarray(sends[k]).reshape(-1)
        lo = int(sum(m[k][:me]))
        parts.append(src[lo:lo + int(m[k][me])])
    dt = np.asarray(sends[0]).dtype
    return np.concatenate(parts).astype(dt, copy=False) if parts else np.empty(0, dtype=dt)


PICK = (0, 1, 3, 5, 257, 4099, 65537)


def tables(n, seed):
    """(name, matrix) pairs: uniform, all zeros, random counts from PICK, one pair carrying almost
    everything, and one rank that sends nothing with another that receives nothing."""
    rng = np.random.default_rng(seed)
    yield "uniform", [[257] * n for _ in range(n)]
    yield "zeros", [[0] * n for _ in range(n)]
    yield "random", [[int(rng.choice(PICK)) for _ in range(n)] for _ in range(n)]
    skew = [[int(rng.integers(0, 4)) for _ in range(n)] for _ in range(n)]
    skew[n - 1][0] = 300001
    yield "one pair", skew
    quiet = [[int(rng.choice(PICK[:5])) for _ in range(n)] for _ in range(n)]
    quiet[0] = [0] * n                    # rank 0 sends nothing
    for i in range(n):
        quiet[i][n - 1] = 0               # rank n-1 receives nothing
    yield "quiet ranks", quiet
