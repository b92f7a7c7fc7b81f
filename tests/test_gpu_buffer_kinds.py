"""GPU tests of collectives whose ranks pass different kinds of buffer in one call (run on an H100:
pytest -m gpu).  The rank processes run _kinds_worker.py: on call i rank r passes the kind
KINDS[(r + i) % len(KINDS)] -- heap views and torch CUDA tensors at aligned and misaligned offsets,
heap and torch on the two sides of one call, pinned host memory from b200mpi_host_alloc and from torch,
and pageable numpy -- and checks every guarded buffer it passed against the oracle after each call.
The enqueue-only entries and a mismatched call run on torch tensors.  A last world runs the chunked
host-slice pipeline with pageable, pinned and registered ranks, and one rank without copy threads, in
the same call.  When the box has fewer GPUs than ranks, the ranks share device 0.

Each rank checks 334 calls in the worlds of 2, 3 and 4 and 214 in the world of 8, and 12 pipelined
calls (6 at 8).  The file takes about 220 s on one H100 80GB HBM3 (700 W power limit), ranks sharing it."""
import os

import pytest

from _kinds_worker import pipe_env
from _launch import assert_world_ok, run_world

pytestmark = pytest.mark.gpu
KINDS_WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_kinds_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}


def world(n, *args, per_rank_env=None, timeout=900):
    res = run_world(n, "kinds", args=list(args), timeout=timeout, env=dict(ENV), per_rank_env=per_rank_env, worker=KINDS_WORKER)
    assert_world_ok(res)
    r0 = res[0]
    print("world of %d: %d calls checked per rank %s, seconds per part %s" % (n, r0["checked"], r0["by_part"], r0["seconds"]))
    return res


@pytest.mark.parametrize("n", [2, 3, 4])
def test_every_collective_across_buffer_kinds(n):
    """Counts 0, 1, EPV+1, 4097 and 65537 for every entry point, the async sequences and the mismatch."""
    world(n)


def test_every_collective_across_buffer_kinds_world_of_8():
    """Counts 1, EPV+1 and 4097."""
    world(8, "--trim", "lean")


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_pipelined_host_slices_with_mixed_pinning(n):
    """Allreduce, Bcast from the first and the last rank and Allgather over several chunks, with the
    pipe and bounce chunks set apart (1 MiB and 256 KiB): every rank must chunk alike whether its
    buffer is bounced, registered, pinned or DMA'd directly.  Before every rank of a multi-rank world
    used the smaller chunk, a pinned rank launched fewer chunks than a pageable one and the launches
    past the first waited for partners that never came."""
    world(n, "--parts", "hostpipe", "--trim", "full" if n < 8 else "lean", per_rank_env=lambda r: pipe_env(n, r))
