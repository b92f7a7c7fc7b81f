"""GPU tests of one-sided communication: WinCreate, Put, Get, Accumulate and the fence (run on an
H100: pytest -m gpu).  Worlds of rank processes drive the public API and the C ABI on guarded windows
and origins and compare every byte with the numpy model of each epoch (_rma_ref.py).  When the box
has fewer GPUs than ranks, the ranks share device 0, so these exercise peer mappings of one GPU, not
NVLink atomics between GPUs."""
import os

import pytest

import _launch
from _launch import assert_world_ok, run_world

pytestmark = pytest.mark.gpu
RMA_WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_rma_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}


@pytest.fixture(autouse=True)
def rma_worker(monkeypatch):
    """The rank processes run _rma_worker.py: _worker.py's entry point plus these scenarios."""
    monkeypatch.setattr(_launch, "WORKER", RMA_WORKER)


def world(n, scenario, timeout=900, env=None):
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, scenario, timeout=timeout, env=e)
    assert_world_ok(res)
    return res


@pytest.mark.parametrize("n", [1, 2, 4, 8])  # 3 ranks: the Accumulate, epoch, error and capped-grid worlds
def test_put_get_dtypes_counts_storages_and_windows(n):
    world(n, "rma")


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_accumulate_overlapping_from_every_rank(n):
    world(n, "rma_accumulate")


@pytest.mark.parametrize("n", [1, 2, 3])
def test_launches_heap_and_epochs(n):
    world(n, "rma_counts")


@pytest.mark.parametrize("n", [1, 3])
def test_consecutive_epochs_between_collectives(n):
    world(n, "rma_epochs")


@pytest.mark.parametrize("n", [3])
def test_past_the_first_grid_pass(n):
    world(n, "rma_capped")


@pytest.mark.parametrize("n", [1, 3])
def test_argument_errors_write_nothing(n):
    world(n, "rma_errors")


def test_staging_that_does_not_fit():
    world(2, "rma_nomem", env={"B200MPI_HEAP_BYTES": str(64 << 20)})


@pytest.mark.parametrize("n", [2, 4])
def test_mismatched_fences_are_reported(n):
    world(n, "rma_mismatch")


def test_64_mib_world_of_4():
    world(4, "rma_large", env={"B200MPI_HEAP_BYTES": str(1 << 30)})
