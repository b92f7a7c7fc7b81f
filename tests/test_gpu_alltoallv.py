"""GPU tests of Alltoallv (run on an H100: pytest -m gpu).  Worlds of rank processes drive the
public API and compare every result bit for bit with the numpy restatement; when the box has fewer
GPUs than ranks, the ranks share device 0."""
import os

import pytest

import _launch
from _launch import assert_world_ok, run_world

pytestmark = pytest.mark.gpu
ALLTOALLV_WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_alltoallv_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}
DTYPES = "u8,f32,f64,i64"


@pytest.fixture(autouse=True)
def alltoallv_worker(monkeypatch):
    """The rank processes run _alltoallv_worker.py: _worker.py's entry point plus these scenarios."""
    monkeypatch.setattr(_launch, "WORKER", ALLTOALLV_WORKER)


def world(n, scenario, *args, timeout=900, env=None):
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, scenario, args=list(args), timeout=timeout, env=e)
    assert_world_ok(res)
    return res


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_alltoallv_tables_dtypes_and_memkinds(n):
    world(n, "alltoallv", "--dtypes", DTYPES, "--kinds", "heap,host")


@pytest.mark.parametrize("n", [2, 3, 4])
def test_alltoallv_unaligned_and_asymmetric_offsets(n):
    world(n, "alltoallv_unaligned")


@pytest.mark.parametrize("n", [2, 4])
def test_alltoallv_mismatched_tables_are_reported(n):
    world(n, "alltoallv_mismatch")


def test_alltoallv_strings_with_learnt_counts_world_of_4():
    world(4, "alltoallv_strings")


def test_alltoallv_large_skewed_world_of_4():
    world(4, "alltoallv_large", env={"B200MPI_HEAP_BYTES": str(1 << 30)})
