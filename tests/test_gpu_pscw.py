"""GPU tests of generalized active-target synchronisation: Post, Start, Complete, Wait and Test (run
on an H100: pytest -m gpu).  Worlds of rank processes run halo exchanges, a star of Accumulates,
disjoint pairs with different epoch counts, the 16-bit counters' wrap in a world of one, every
argument and state error, timeouts, fences against open epochs and the reuse of window cells, with
guarded windows checked byte for byte.  When the box has fewer GPUs than ranks, the ranks share
device 0, so these exercise peer mappings of one GPU, not NVLink between GPUs."""
import os

import pytest

import _launch
from _launch import assert_world_ok, run_world

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_pscw_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}


@pytest.fixture(autouse=True)
def pscw_worker(monkeypatch):
    """The rank processes run _pscw_worker.py: _worker.py's entry point plus these scenarios."""
    monkeypatch.setattr(_launch, "WORKER", WORKER)


def world(n, scenario, timeout=600):
    assert_world_ok(run_world(n, scenario, timeout=timeout, env=dict(ENV)))


@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_ring_halo_exchange(n):
    world(n, "pscw_halo")


@pytest.mark.parametrize("n", [1, 4, 8])
def test_star_accumulate_is_exact(n):
    world(n, "pscw_star")


def test_disjoint_pairs_synchronise_alone():
    world(4, "pscw_disjoint")


@pytest.mark.parametrize("n", [1, 3])
def test_one_launch_no_epoch_no_heap(n):
    world(n, "pscw_counts")


@pytest.mark.parametrize("n", [1, 3])
def test_groups_with_this_rank_and_counter_wrap(n):
    world(n, "pscw_self")


@pytest.mark.parametrize("n", [1, 3])
def test_argument_and_state_errors_launch_nothing(n):
    world(n, "pscw_errors")


def test_start_and_wait_time_out_and_then_succeed():
    world(2, "pscw_timeout")


def test_start_keeps_the_posts_that_arrived_before_a_timeout():
    world(3, "pscw_partial")


@pytest.mark.parametrize("n", [1, 2, 4])
def test_fence_and_free_against_an_open_epoch(n):
    world(n, "pscw_fence")


@pytest.mark.parametrize("n", [1, 3])
def test_cells_of_created_and_freed_windows_start_clear(n):
    world(n, "pscw_cells")
