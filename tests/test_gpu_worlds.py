"""GPU parity tests (run on an H100: pytest -m gpu).  Every test launches a world of rank
processes through the gompirun-style launcher and drives the product through the public API /
C ABI; results are compared with the CPU oracle on the same seeded inputs.  When the box has fewer
GPUs than ranks, ranks share device 0 (the kernels and the peer mappings are the same; the GPU
time-slices between the processes)."""
import os
import subprocess

import pytest

from _launch import assert_world_ok, run_world

pytestmark = pytest.mark.gpu
ENV = {"B200MPI_WATCHDOG_S": "90"}


def ngpus():
    try:
        return subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout.count("GPU ")
    except Exception:  # noqa: BLE001
        return 0


def world(n, scenario, *args, timeout=900, env=None, per_rank_env=None):  # generous: the pod's host CPUs are shared, a world of 8 Python ranks can start slowly
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, scenario, args=list(args), timeout=timeout, env=e, per_rank_env=per_rank_env)
    assert_world_ok(res)
    return res


def need_gpus(k, what):
    have = ngpus()
    if have < k:
        pytest.skip("%s needs >= %d GPUs with NVLink/NVLS between them; this box has %d (ranks sharing one GPU cannot bind a multicast object)" % (what, k, have))
    return have


def assert_nothing_skipped(results):
    sk = sorted({x for r in results for x in r.get("skipped", [])})
    assert not sk, "the switch paths did not run: %s" % sk


def test_smoke_world_of_1_and_2():
    r1 = world(1, "smoke")
    assert r1[0]["device"] == 0
    r2 = world(2, "smoke")
    assert all(r["launches"] >= 1 for r in r2)


@pytest.mark.parametrize("n", [1, 2])
def test_collectives_small_sizes_all_algorithms(n):
    world(n, "collectives")


def test_collectives_world_of_4():
    world(4, "collectives", "--sizes", "0,1,5,257,65537", "--kinds", "heap")


def test_collectives_world_of_3_generic_kernels():
    world(3, "collectives", "--sizes", "3,257,4099", "--kinds", "heap,host")


def test_collectives_world_of_8():
    world(8, "collectives", "--sizes", "1,257,40001", "--kinds", "heap", "--dtypes", "f32,i64", timeout=900)


@pytest.mark.parametrize("n", [2, 4])
def test_edge_values_and_identical_results(n):
    world(n, "edge_values")


def test_unaligned_and_asymmetric_offsets():
    world(2, "unaligned")
    world(4, "unaligned")


def bounce_worlds(per_rank_env=None):
    # examples/bounce: the reference's size ladder (bounce.go:33) up to 1e7 bytes + the 1 MiB float64
    # point; with 1 MiB chunks the largest sizes wrap the 4-region staging ring
    world(2, "p2p", "--sizes", "0,1,10,100,1000,10000,100000,1000000,10000000,1048576", env={"B200MPI_STAGE_CHUNK": str(1 << 20)},
          per_rank_env=per_rank_env)
    world(4, "p2p", "--sizes", "0,8,4096,1048576", per_rank_env=per_rank_env)


def test_bounce_send_receive():
    bounce_worlds()


@pytest.mark.parametrize("fast_ranks", ["all", "rank0"])
def test_bounce_send_receive_mapped_bounce(fast_ranks):
    """The mapped-bounce path (host slices of at most 4 MiB) is off by default when ranks share a GPU,
    so it is forced on: on every rank, and on rank 0 only, where a bounce sender meets a ring receiver
    and a ring sender meets a bounce receiver."""
    bounce_worlds(lambda r: {"B200MPI_P2P_FAST": "1" if fast_ranks == "all" or r == 0 else "0"})


def test_send_receive_device_memory_outside_the_heap():
    # torch CUDA tensors (memkind DEVICE, not in the heap), over several 1 MiB staging chunks
    world(2, "p2p_torch", env={"B200MPI_STAGE_CHUNK": str(1 << 20)})


@pytest.mark.parametrize("n", [1, 2, 4])
def test_helloworld(n):
    world(n, "helloworld")


def test_concurrent_tags_and_duplicate_tag():
    world(2, "tags")


@pytest.mark.parametrize("n", [1, 2])
def test_caller_stream_async_calls_and_timer(n):
    world(n, "stream")


def test_mismatched_collectives_are_reported_not_hung():
    world(2, "mismatch")
    world(4, "mismatch")


@pytest.mark.parametrize("n", [2, 4])
def test_ll_allreduce(n):
    """Barrier-free LL allreduce (the small-message default on real multi-GPU worlds): rank-order
    results, bit-exact; device pointers and host slices (mapped pinned bounce, one kernel)."""
    world(n, "collectives", "--algos", "ll", "--sizes", "0,1,2,3,257,4097,8192,40000", "--kinds", "heap,host")


@pytest.mark.parametrize("n", [2, 3, 4])
def test_reduce_scatter_reduce_alltoall(n):
    world(n, "newcolls", "--sizes", "0,1,5,257,4099,70001")


def test_reduce_scatter_reduce_alltoall_world_of_8():
    world(8, "newcolls", "--sizes", "3,4099", "--kinds", "heap", "--dtypes", "f32,i64", timeout=900)


@pytest.mark.parametrize("n", [1, 2, 4])
def test_host_slice_pipeline_pageable_and_pinned(n):
    world(n, "hostpipe", "--sizes", "16385,300001", "--dtypes", "f32,i64" if n == 4 else "f32,f64,i64")


def test_isend_wait():
    world(2, "isend")
    world(4, "isend")
    world(2, "isend", env={"B200MPI_P2P_FAST": "1"})  # host Isends of at most 4 MiB go through the mapped bounce


def test_send_timeout_withdraws_the_post():
    world(2, "sendtimeout")


def test_switch_paths_on_real_nvlink():
    """NVLS / hybrid allreduce, NVLS allgather, bcast and reduce-scatter, and LL over real NVLink.
    They cannot run when ranks share one GPU: shown as SKIPPED there, never as passed."""
    have = need_gpus(2, "multimem (NVLS) kernels")
    n = 8 if have >= 8 else 4 if have >= 4 else 2
    res = world(n, "collectives", "--algos", "nvls,hybrid,ll", "--sizes", "1,257,4096,40001,1048577", "--kinds", "heap", timeout=900,
                env={"B200MPI_HEAP_BYTES": str(512 << 20)})
    assert all(r["nvls"] for r in res), "multicast mapping was not set up on a multi-GPU box"
    assert_nothing_skipped(res)
    res = world(n, "newcolls", "--sizes", "1,4099,262144", "--kinds", "heap", timeout=900, env={"B200MPI_HEAP_BYTES": str(512 << 20)})
    assert_nothing_skipped(res)


def test_full_size_points():
    """BASELINE.json sizes: Allgather int64 1 Mi per rank x 8 ranks bit-exact; Allreduce f32 at 16 Mi
    elements (64 MiB) with every algorithm; bounce 1 MiB float64 is covered above."""
    world(8, "fullsize", "--what", "allgather", timeout=900, env={"B200MPI_HEAP_BYTES": str(512 << 20)})
    world(2, "fullsize", "--what", "allreduce", timeout=900, env={"B200MPI_HEAP_BYTES": str(1 << 30)})


def test_flag_scrub_between_collectives():
    """Every kScrubEvery-th launch is preceded by scrub_kernel (rewrites every barrier slot so that the
    wrap-safe flag comparisons stay sound on long jobs).  B200MPI_SCRUB_EVERY=4 makes that every 4th
    launch here; results must be unaffected.  (Last in the file: written after the round's GPU budget
    was spent, so its first run is the driver's.)"""
    world(2, "collectives", "--sizes", "1,257,65537", "--kinds", "heap", "--dtypes", "f32", env={"B200MPI_SCRUB_EVERY": "4"})
    world(4, "collectives", "--sizes", "257,4099", "--kinds", "heap", "--dtypes", "i64", env={"B200MPI_SCRUB_EVERY": "4"})

