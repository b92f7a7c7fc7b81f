"""GPU tests of AllreduceLoc and ReduceLoc, MAXLOC / MINLOC (run on an H100: pytest -m gpu).  Worlds of
rank processes drive the public API and the C ABI on guarded buffers and compare every result with
the C oracle byte for byte, padding included; when the box has fewer GPUs than ranks, the ranks
share device 0."""
import os

import pytest

import _launch
from _launch import assert_world_ok, run_world
from test_gpu_wrap import EPOCH_WRAP, start_below

pytestmark = pytest.mark.gpu
LOC_WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_loc_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}


@pytest.fixture(autouse=True)
def loc_worker(monkeypatch):
    """The rank processes run _loc_worker.py: _worker.py's entry point plus these scenarios."""
    monkeypatch.setattr(_launch, "WORKER", LOC_WORKER)


def world(n, scenario, *args, timeout=900, env=None):
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, scenario, args=list(args), timeout=timeout, env=e)
    assert_world_ok(res)
    return res


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_loc_dtypes_ops_counts_storages_and_roots(n):
    world(n, "loc")


@pytest.mark.parametrize("n", [2, 3])
def test_loc_past_the_first_grid_pass(n):
    world(n, "loc_capped")


@pytest.mark.parametrize("n", [2, 4])
def test_loc_mismatches_are_reported(n):
    world(n, "loc_mismatch")


@pytest.mark.parametrize("n", [2, 3])
def test_loc_across_the_epoch_wrap(n):
    res = world(n, "loc_wrap", env={"B200MPI_SCRUB_EVERY": "4", "B200MPI_EPOCH_START": start_below(EPOCH_WRAP)})
    for r in res:
        assert r["epoch_first"] >= 1 << 31 and r["epoch_last"] < 1 << 31, r  # the 32-bit epoch wrapped during the run


def test_loc_64_mib_world_of_4():
    world(4, "loc_large", env={"B200MPI_HEAP_BYTES": str(1 << 30)})


@pytest.mark.parametrize("n", [1, 3, 4])
def test_minloc_names_the_rank_whose_point_bcast_delivers(n):
    world(n, "loc_best_point")
