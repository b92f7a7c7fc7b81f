"""GPU tests of ReduceScatterv (run on an H100: pytest -m gpu).  Worlds of rank processes drive the
public API and compare every rank's block bit for bit with the rank-order reduction of the C oracle;
when the box has fewer GPUs than ranks, the ranks share device 0."""
import os

import pytest

import _launch
from _launch import assert_world_ok, run_world
from test_gpu_wrap import EPOCH_WRAP, start_below

pytestmark = pytest.mark.gpu
RSV_WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_rsv_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}


@pytest.fixture(autouse=True)
def rsv_worker(monkeypatch):
    """The rank processes run _rsv_worker.py: _worker.py's entry point plus these scenarios."""
    monkeypatch.setattr(_launch, "WORKER", RSV_WORKER)


def world(n, scenario, *args, timeout=900, env=None):
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, scenario, args=list(args), timeout=timeout, env=e)
    assert_world_ok(res)
    return res


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_reduce_scatterv_dtypes_ops_tables_and_memkinds(n):
    world(n, "rsv")


@pytest.mark.parametrize("n", [2, 3, 4])
def test_reduce_scatterv_writes_exactly_its_recv(n):
    world(n, "rsv_footprint")


@pytest.mark.parametrize("n", [2, 4])
def test_reduce_scatterv_mismatches_are_reported(n):
    world(n, "rsv_mismatch")


@pytest.mark.parametrize("n", [2, 3])
def test_reduce_scatterv_across_the_epoch_wrap(n):
    res = world(n, "rsv_wrap", env={"B200MPI_SCRUB_EVERY": "4", "B200MPI_EPOCH_START": start_below(EPOCH_WRAP)})
    for r in res:
        assert r["epoch_first"] >= 1 << 31 and r["epoch_last"] < 1 << 31, r  # the 32-bit epoch wrapped during the run


@pytest.mark.parametrize("n", [2, 3, 4])
def test_sharded_allreduce_equals_two_shot_allreduce(n):
    world(n, "rsv_sharded_allreduce")


def test_reduce_scatterv_64_mib_world_of_4():
    world(4, "rsv_large", env={"B200MPI_HEAP_BYTES": str(1 << 30)})
