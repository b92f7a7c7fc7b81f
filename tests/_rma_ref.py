"""numpy model of one fence epoch of one-sided communication (b200mpi_put / _get / _accumulate).

Windows are byte images, one per rank.  A Get reads what the target's window held at the fence that
opened the epoch; Puts and Accumulates land in the images the next fence publishes.  Accumulates are
applied one after another in call order: the tests choose values for which every order gives the
same bytes (exactly representable sums).  The element rules are those of include/b200mpi.h: i64 SUM
wraps, i64 MAX / MIN are exact, f32 SUM flushes subnormal inputs and results to zero of the same
sign."""
import numpy as np

SUM, MAX, MIN = 0, 1, 2
F32_MIN_NORMAL = np.float32(np.finfo(np.float32).tiny)


def ftz32(x):
    """Subnormal f32 values become zero of the same sign."""
    x = np.asarray(x, dtype=np.float32)
    return np.where(np.abs(x) < F32_MIN_NORMAL, np.copysign(np.float32(0), x), x).astype(np.float32)


def combine(a, b, op):
    """target element values a updated by contributions b (same dtype)."""
    a, b = np.asarray(a), np.asarray(b)
    dt = a.dtype
    if op == SUM:
        if dt == np.int64:
            return (a.view(np.uint64) + b.view(np.uint64)).view(np.int64)  # Go int64 wrap
        if dt == np.float32:
            return ftz32(ftz32(a) + ftz32(b))
        return (a + b).astype(dt)
    if op == MAX:
        return np.where(b > a, b, a).astype(dt)
    if op == MIN:
        return np.where(b < a, b, a).astype(dt)
    raise ValueError(op)


class Epoch:
    """One fence epoch over `windows` (uint8 arrays, one per rank; copied)."""

    def __init__(self, windows):
        self.start = [np.array(w, dtype=np.uint8, copy=True) for w in windows]
        self.now = [w.copy() for w in self.start]

    @staticmethod
    def _span(win, dt, disp, count):
        es = np.dtype(dt).itemsize
        lo, hi = disp * es, (disp + count) * es
        assert hi <= win.size, "outside the window"
        return lo, hi

    def put(self, origin, target, disp):
        origin = np.ascontiguousarray(origin)
        lo, hi = self._span(self.now[target], origin.dtype, disp, origin.size)
        self.now[target][lo:hi] = origin.view(np.uint8)

    def get(self, dt, count, target, disp):
        lo, hi = self._span(self.start[target], dt, disp, count)
        return self.start[target][lo:hi].copy().view(dt)

    def accumulate(self, origin, target, disp, op):
        origin = np.ascontiguousarray(origin)
        lo, hi = self._span(self.now[target], origin.dtype, disp, origin.size)
        cur = self.now[target][lo:hi].copy().view(origin.dtype)
        self.now[target][lo:hi] = combine(cur, origin, op).view(np.uint8)

    def fence(self):
        """The windows every rank sees after the closing fence."""
        return [w.copy() for w in self.now]
