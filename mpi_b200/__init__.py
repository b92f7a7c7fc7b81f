"""mpi_b200 -- H100-native transport behind the btracey/mpi API.

`import mpi_b200 as mpi` gives the reference's package surface (mpi.go) over libb200mpi.so:
Init, Finalize, Rank, Size, Send, Receive (+ Recv, Bcast, Allreduce, Allgather, Barrier,
ReduceScatter, Reduce, Alltoall, Gather, Scatter, Gatherv, Scatterv, Allgatherv, Alltoallv,
Scan, Exscan, ReduceScatterv, AllreduceLoc, ReduceLoc (MAXLOC / MINLOC over the LOC_F32, LOC_F64
and LOC_I64 pair dtypes), WinCreate (one-sided Put, Get and Accumulate through a Win, and the
passive-target Lock, Unlock, GetAccumulate, FetchAndOp and CompareAndSwap, and the generalized
active-target Post, Start, Complete, Wait and Test), Isend/Wait).
The shared library (mpi_b200/lib/libb200mpi.so, built by mpi_b200/csrc/Makefile) is loaded on
first use; nothing here computes or moves payload bytes in Python.
"""
from ._lib import LIB_PATH, load  # noqa: F401
from .api import (  # noqa: F401
    LOC_F32, LOC_F64, LOC_I64, LOCK_EXCLUSIVE, LOCK_SHARED, MAX, MIN, NO_OP, REPLACE, SUM, Alloc, Allgather, Allgatherv, Allreduce, AllreduceLoc, Alltoall, Alltoallv,
    Barrier, Bcast, Cuda, DeviceSlice, Exscan, Finalize, Gather, Gatherv, Init, Interface, Isend, MpiError, Rank, Raw,
    Receive, Recv, Reduce, ReduceLoc, ReduceScatter, ReduceScatterv, Register, Scan, Scatter, Scatterv, Send, Size,
    TagExists, Wait, Win, WinCreate)
from . import flags  # noqa: F401
