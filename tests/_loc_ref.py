"""MAXLOC / MINLOC restated in numpy -- TEST INFRASTRUCTURE, independent of loc_oracle.c.

A pair is {val, loc} in a LOC_F32 / LOC_F64 / LOC_I64 array (16 bytes; an f32 value is followed by
4 padding bytes).  combine(a, b, op) is one step of the rank-order fold, a holding the lower ranks:
b's pair replaces a's when b's value is better, or equal with a smaller loc.  Floats compare as IEEE
(-0 == +0) except that NaN beats every number under both ops and equals every NaN.  Pairs move as
raw 16-byte words, padding included."""
import numpy as np

import mpi_b200 as mpi

MAX, MIN = mpi.MAX, mpi.MIN
LOC = {"f32": mpi.LOC_F32, "f64": mpi.LOC_F64, "i64": mpi.LOC_I64}


def words(x):
    """The pairs of x as (count, 2) uint64 words: value bits (and padding), loc."""
    return np.ascontiguousarray(x).reshape(-1).view(np.uint64).reshape(-1, 2)


def concat(xs):
    """np.concatenate of pair arrays, padding kept (numpy drops it when it copies structured elements)."""
    return np.concatenate([words(x) for x in xs]).reshape(-1).view(xs[0].dtype)


def pairs(dt, vals, locs, pads=None):
    """A pair array of dtype dt; pads (f32 only) are the 4 padding bytes of each pair as a uint32."""
    dt = np.dtype(dt)
    vals = np.asarray(vals, dtype=dt["val"]).reshape(-1)
    w = np.zeros((vals.size, 2), dtype=np.uint64)
    if dt["val"].itemsize == 4:
        w[:, 0] = vals.view(np.uint32).astype(np.uint64)
        if pads is not None:
            w[:, 0] |= np.asarray(pads, dtype=np.uint64) << np.uint64(32)
    else:
        w[:, 0] = vals.view(np.uint64)
    w[:, 1] = np.asarray(locs, dtype=np.int64).reshape(-1).view(np.uint64)
    return w.reshape(-1).view(dt)


def replaces(a, b, op):
    """Per pair: does b's pair replace a's?"""
    x, y = a["val"], b["val"]
    with np.errstate(invalid="ignore"):
        cmp = (y > x) if op == MAX else (y < x)
        eq = x == y
    if x.dtype.kind == "f":
        xn, yn = np.isnan(x), np.isnan(y)
        better = ~xn & (yn | cmp)
        equal = np.where(xn, yn, ~yn & eq)
    else:
        better, equal = cmp, eq
    return better | (equal & (b["loc"] < a["loc"]))


def combine(a, b, op):
    take = replaces(a, b, op)
    return np.where(take[:, None], words(b), words(a)).reshape(-1).view(a.dtype)


def fold_left(xs, op):
    acc = xs[0]
    for x in xs[1:]:
        acc = combine(acc, x, op)
    return acc


def fold_right(xs, op):
    acc = xs[-1]
    for x in reversed(xs[:-1]):
        acc = combine(x, acc, op)
    return acc


def fold_tree(xs, op):
    """((x0 x1)(x2 x3))((x4 x5)(x6 x7)): neighbours combined level by level, lower ranks on the left."""
    level = list(xs)
    while len(level) > 1:
        nxt = [combine(level[i], level[i + 1], op) for i in range(0, len(level) - 1, 2)]
        if len(level) % 2:
            nxt.append(level[-1])
        level = nxt
    return level[0]


def allreduce_loc_np(xs, op):
    return fold_left([np.ascontiguousarray(x).reshape(-1) for x in xs], op)


def same(a, b):
    """Byte for byte, padding included."""
    return a.dtype == b.dtype and a.size == b.size and np.array_equal(words(a), words(b))


def tie_heavy(dn, n, count, seed):
    """Every rank's pairs drawn from small sets, so that equal values and equal locs are frequent:
    floats from {-inf, -1.5, -0, +0, 1.5, inf, NaN (payload naming the rank)}, i64 from
    {INT64_MIN, -1, 0, 1, INT64_MAX}; locs from {-3, 0, 2, 5}; f32 padding random."""
    dt = LOC[dn]
    rng = np.random.default_rng([0x10C, seed])
    out = []
    for r in range(n):
        if dn == "i64":
            pool = np.array([np.iinfo(np.int64).min, -1, 0, 1, np.iinfo(np.int64).max], dtype=np.int64)
            vals = pool[rng.integers(0, pool.size, size=count)]
        else:
            vt = np.float32 if dn == "f32" else np.float64
            pool = np.array([-np.inf, -1.5, -0.0, 0.0, 1.5, np.inf], dtype=vt)
            vals = pool[rng.integers(0, pool.size, size=count)]
            nan = rng.random(count) < 0.12
            payload = (0x7FC00000 | (0x100 + r)) if dn == "f32" else (0x7FF8000000000000 | (0x100 + r))
            bits = vals.view(np.uint32 if dn == "f32" else np.uint64).copy()
            bits[nan] = payload
            vals = bits.view(vt)
        locs = np.array([-3, 0, 2, 5], dtype=np.int64)[rng.integers(0, 4, size=count)]
        pads = rng.integers(0, 1 << 32, size=count, dtype=np.uint64) if dn == "f32" else None
        out.append(pairs(dt, vals, locs, pads))
    return out
