"""GPU tests of the passive-target calls: Lock, Unlock, GetAccumulate, FetchAndOp and CompareAndSwap
(run on an H100: pytest -m gpu).  Worlds of rank processes take tickets, hold elections, swap values,
update records under locks and check every element rule against the numpy model (_rma_atomic_ref.py)
byte for byte, on guarded windows, origins and results.  When the box has fewer GPUs than ranks, the
ranks share device 0, so these exercise atomics through peer mappings of one GPU, not NVLink atomics
between GPUs."""
import os

import pytest

import _launch
from _launch import assert_world_ok, run_world

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_rma_atomic_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}


@pytest.fixture(autouse=True)
def rma_atomic_worker(monkeypatch):
    """The rank processes run _rma_atomic_worker.py: _worker.py's entry point plus these scenarios."""
    monkeypatch.setattr(_launch, "WORKER", WORKER)


def world(n, scenario, timeout=600):
    assert_world_ok(run_world(n, scenario, timeout=timeout, env=dict(ENV)))


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_tickets_are_every_number_once(n):
    world(n, "ra_tickets")


@pytest.mark.parametrize("n", [1, 3, 8])
def test_election_has_one_winner_per_cell(n):
    world(n, "ra_election")


@pytest.mark.parametrize("n", [1, 4])
def test_swap_chain_is_a_permutation(n):
    world(n, "ra_swap")


@pytest.mark.parametrize("n", [1, 2])
def test_element_rules_against_the_model(n):
    world(n, "ra_rules")


@pytest.mark.parametrize("n", [1, 2, 4, 8])
def test_locks_exclude_and_publish(n):
    world(n, "ra_mutex")


@pytest.mark.parametrize("n", [1, 3])
def test_one_launch_no_epoch_no_heap(n):
    world(n, "ra_counts")


@pytest.mark.parametrize("n", [1, 3])
def test_argument_errors_write_nothing(n):
    world(n, "ra_errors")


@pytest.mark.parametrize("n", [1, 2, 4])
def test_fence_against_a_held_lock(n):
    world(n, "ra_fence_locked")


def test_lock_times_out_and_then_succeeds():
    world(2, "ra_timeout")


@pytest.mark.parametrize("n", [1, 3])
def test_lock_cells_of_created_and_freed_windows(n):
    world(n, "ra_cells")
