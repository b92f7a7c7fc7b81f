"""GPU tests of what every collective writes (run on an H100: pytest -m gpu).  The rank processes run
_footprint_worker.py: every buffer is a view with guard bytes on both sides, at aligned, symmetric,
per-rank and send/recv-split misalignments, and every rank checks the whole allocation of every
buffer it passed after each call -- guards and out-of-place sends unchanged, destinations bit-exact
against the oracle in the order of the kernel that ran, MAX and MIN over signed and special values
included.  When the box has fewer GPUs than ranks, the ranks share device 0."""
import os

import pytest

from _launch import assert_world_ok, run_world
from test_gpu_worlds import assert_nothing_skipped, need_gpus

pytestmark = pytest.mark.gpu
FOOTPRINT_WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_footprint_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}
P2P_PARTS = "allreduce,reduce,reduce_scatter,bytes,v,p2p"


def world(n, *args, env=None, timeout=900):
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, "footprint", args=list(args), timeout=timeout, env=e, worker=FOOTPRINT_WORKER)
    assert_world_ok(res)
    r0 = res[0]
    print("world of %d: %d calls checked per rank %s, seconds per part %s" % (n, r0["checked"], r0["by_part"], r0["seconds"]))
    return res


@pytest.mark.parametrize("n", [2, 3, 4, 6])
def test_every_collective_writes_exactly_its_destination(n):
    """Every count of counts_for in worlds of 2-4; in the world of 6 without EPV-1 and 257."""
    world(n, "--parts", P2P_PARTS, "--trim", "full" if n <= 4 else "lean")


def test_every_collective_writes_exactly_its_destination_world_of_8():
    """1, EPV+1 and one grid pass +-1 vector per kernel."""
    world(8, "--parts", P2P_PARTS, "--trim", "edges")


def test_switch_paths_write_exactly_their_destination():
    """NVLS and hybrid Allreduce (i64 MAX / MIN included), the NVLS Reduce with asymmetric offsets,
    ReduceScatter and both NVLS Bcasts.  They cannot run when ranks share one GPU: shown as SKIPPED
    there, never as passed."""
    have = need_gpus(2, "multimem (NVLS) kernels")
    n = 8 if have >= 8 else 4 if have >= 4 else 2
    res = world(n, "--parts", "nvls", env={"B200MPI_HEAP_BYTES": str(512 << 20)})
    assert all(r["nvls"] for r in res), "multicast mapping was not set up on a multi-GPU box"
    assert_nothing_skipped(res)
