"""Oracle of AllreduceLoc and ReduceLoc (MAXLOC / MINLOC) -- TEST INFRASTRUCTURE.

ctypes front end of loc_oracle.c, compiled on first use into a private temporary directory so the
tree is never written.  Its independent numpy restatement is _loc_ref.py."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from mpi_b200.api import _LOC2DT

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "loc_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="b200mpi-loc-oracle-"), "libloc_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-std=gnu11", "-shared", "-o", so, _SRC])
        h = ctypes.CDLL(so)
        c = ctypes
        h.oracle_allreduce_loc.argtypes = [c.c_int, c.c_int, c.c_int, c.c_size_t, c.POINTER(c.c_void_p), c.c_void_p]
        _lib = h
    return _lib


def allreduce_loc(inputs, op):
    """inputs[r]: rank r's pair array (a LOC_* dtype); returns the winning pairs, bytes as the oracle
    copied them.  op: L.MAX (MAXLOC) or L.MIN (MINLOC)."""
    arrs = [np.ascontiguousarray(a).reshape(-1) for a in inputs]
    dt = arrs[0].dtype
    n, count = len(arrs), arrs[0].size
    out = np.zeros(count, dtype=dt)
    ptrs = (ctypes.c_void_p * n)(*[a.ctypes.data for a in arrs])
    if lib().oracle_allreduce_loc(_LOC2DT[dt], int(op), n, count, ptrs, out.ctypes.data):
        raise ValueError("oracle_allreduce_loc: bad arguments")
    return out
