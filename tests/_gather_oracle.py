"""Oracle of Gather, Scatter, Gatherv, Scatterv and Allgatherv -- TEST INFRASTRUCTURE.

ctypes front end of gather_oracle.c (compiled on first use into a private temporary directory, so
the tree is never written) plus an independent numpy twin of the same semantics."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gather_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="b200mpi-gather-oracle-"), "libgather_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-std=gnu11", "-shared", "-o", so, _SRC])
        L = ctypes.CDLL(so)
        c = ctypes
        L.oracle_gatherv.argtypes = [c.c_size_t, c.c_int, c.POINTER(c.c_size_t), c.POINTER(c.c_void_p), c.c_void_p]
        L.oracle_scatterv.argtypes = [c.c_size_t, c.c_int, c.c_int, c.POINTER(c.c_size_t), c.c_void_p, c.c_void_p]
        _lib = L
    return _lib


def gatherv(inputs):
    """inputs[r] holds rank r's block (any length); returns root's recv: the blocks packed in rank order."""
    n = len(inputs)
    arrs = [np.ascontiguousarray(a).reshape(-1) for a in inputs]
    dt = arrs[0].dtype
    counts = (ctypes.c_size_t * n)(*[a.size for a in arrs])
    out = np.empty(sum(a.size for a in arrs), dtype=dt)
    ptrs = (ctypes.c_void_p * n)(*[a.ctypes.data for a in arrs])
    if lib().oracle_gatherv(dt.itemsize, n, counts, ptrs, out.ctypes.data):
        raise ValueError("oracle_gatherv: bad arguments")
    return out


def scatterv(root_send, counts, me):
    """root_send holds sum(counts) elements; returns what rank `me` receives."""
    n = len(counts)
    src = np.ascontiguousarray(root_send).reshape(-1)
    out = np.empty(int(counts[me]), dtype=src.dtype)
    table = (ctypes.c_size_t * n)(*[int(c) for c in counts])
    if lib().oracle_scatterv(src.dtype.itemsize, n, me, table, src.ctypes.data, out.ctypes.data):
        raise ValueError("oracle_scatterv: bad arguments")
    return out


# ---- numpy twin (independent restatement used to cross-check the C oracle) --------------------
def gatherv_np(inputs):
    return np.concatenate([np.asarray(a).reshape(-1) for a in inputs])


def scatterv_np(root_send, counts, me):
    lo = int(sum(counts[:me]))
    return np.array(np.asarray(root_send).reshape(-1)[lo:lo + int(counts[me])], copy=True)
