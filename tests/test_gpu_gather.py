"""GPU tests of Gather, Scatter, Gatherv, Scatterv and Allgatherv (run on an H100: pytest -m gpu).
Worlds of rank processes drive the public API and compare every result bit for bit with the CPU
oracle; when the box has fewer GPUs than ranks, the ranks share device 0."""
import os

import pytest

import _launch
from _launch import assert_world_ok, run_world

pytestmark = pytest.mark.gpu
GATHER_WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_gather_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}
COUNTS = "0,1,3,5,257,4099,65537"
DTYPES = "u8,f32,f64,i64"


@pytest.fixture(autouse=True)
def gather_worker(monkeypatch):
    """The rank processes run _gather_worker.py: _worker.py's entry point plus these scenarios."""
    monkeypatch.setattr(_launch, "WORKER", GATHER_WORKER)


def world(n, scenario, *args, timeout=900, env=None):
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, scenario, args=list(args), timeout=timeout, env=e)
    assert_world_ok(res)
    return res


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_gather_scatter_every_root_dtype_and_memkind(n):
    world(n, "gather", "--sizes", COUNTS, "--dtypes", DTYPES, "--kinds", "heap,host")


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_v_tables_zero_odd_and_skewed(n):
    world(n, "gatherv", "--dtypes", DTYPES, "--kinds", "heap,host")


@pytest.mark.parametrize("n", [2, 4])
def test_unaligned_and_asymmetric_offsets(n):
    world(n, "gather_unaligned")


@pytest.mark.parametrize("n", [2, 4])
def test_mismatched_tables_and_roots_are_reported(n):
    world(n, "gather_mismatch")


def test_strings_of_different_lengths_world_of_4():
    world(4, "gather_strings")


def test_gather_full_size_world_of_4():
    world(4, "gather_fullsize", env={"B200MPI_HEAP_BYTES": str(1 << 30)})
