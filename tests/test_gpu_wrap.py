"""GPU tests of the 32-bit counters at their wraps (run on an H100: pytest -m gpu).  Worlds start a few
launches below a boundary through the test hooks B200MPI_EPOCH_START / B200MPI_LL_SEQ_START, with a
scrub every 4th launch so that scrubs land on both sides of it, and compare every result with the
oracle.  When the box has fewer GPUs than ranks, the ranks share device 0."""
import os

import pytest

import _launch
from _launch import assert_world_ok, run_world
from mpi_b200 import _lib as L
from test_gpu_worlds import assert_nothing_skipped, need_gpus

pytestmark = pytest.mark.gpu
WRAP_WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_wrap_worker.py")
STRIDE = 4096
EPOCH_WRAP = 1 << 20   # epoch index of the first launch after the epoch wraps (start value 1)
RING_WRAP = 1 << 17    # epoch index where the ring step counters (epoch * 8) wrap


def start_below(index, strides=12):
    """B200MPI_EPOCH_START a few launches below epoch index `index`."""
    return str(((index - strides) * STRIDE + 1) % (1 << 32))


ENV = {"B200MPI_WATCHDOG_S": "90", "B200MPI_SCRUB_EVERY": "4"}


@pytest.fixture(autouse=True)
def wrap_worker(monkeypatch):
    """The rank processes run _wrap_worker.py: _worker.py's entry point plus these scenarios."""
    monkeypatch.setattr(_launch, "WORKER", WRAP_WORKER)


def world(n, scenario, *args, env=None, timeout=900, boundary=EPOCH_WRAP):
    e = dict(ENV)
    e["B200MPI_EPOCH_START"] = start_below(boundary)
    if env:
        e.update(env)
    res = run_world(n, scenario, args=list(args), timeout=timeout, env=e)
    assert_world_ok(res)
    return res


# (family, world size, variants "dtype:kind:count:in|out" run just before and just after the wrap)
FAMILY_CASES = [
    ("oneshot", 2, "f32:heap:257:in,f64:host:1001:out,i64:heap:4099:in"),
    ("oneshot", 4, "f32:heap:5:out,i64:heap:65537:in"),
    ("oneshot", 3, "f32:heap:4099:in,f64:host:257:out,i64:heap:3:in"),
    ("twoshot", 2, "f32:heap:65537:out,i64:host:257:in,f64:heap:4099:in"),
    ("twoshot", 4, "f64:heap:4099:out,f32:heap:70001:in"),
    ("twoshot", 3, "i64:heap:4099:in,f32:host:257:out"),
    ("smem", 2, "f32:heap:70001:in,f64:host:4099:out"),
    ("smem", 4, "i64:heap:65537:out,f32:heap:257:in"),
    ("ring", 2, "f32:heap:65537:in,i64:host:1001:out"),
    ("ring", 4, "f64:heap:4099:out,f32:heap:257:in"),
    ("ring", 3, "i64:heap:70001:in,f32:heap:5:out"),
    ("bcast_oneshot", 2, "u8:heap:1501:out,f64:host:257:out"),
    ("bcast_oneshot", 4, "f32:heap:65537:out,i64:heap:3:out"),
    ("bcast_twoshot", 2, "i64:heap:4099:out,u8:host:70001:out"),
    ("bcast_twoshot", 4, "f32:heap:70001:out,u8:heap:1501:out"),
    ("allgather_push", 2, "u8:heap:1501:out,f32:host:4099:out"),
    ("allgather_push", 4, "i64:heap:257:out,f64:heap:65537:out"),
    ("allgather_ring", 2, "f64:heap:4099:out,u8:host:257:out"),
    ("allgather_ring", 4, "u8:heap:70001:out,f32:heap:5:out"),
    ("reduce_scatter", 2, "f32:heap:4099:out,i64:host:257:out"),
    ("reduce_scatter", 4, "f64:heap:1001:out,f32:heap:5:out"),
    ("reduce", 2, "i64:heap:4099:out,f32:host:257:out"),
    ("reduce", 4, "f64:heap:70001:out,f32:heap:5:out"),
    ("alltoall", 2, "f64:heap:1001:out,i64:host:3:out"),
    ("alltoall", 4, "f32:heap:4099:out,i64:heap:257:out"),
    ("gatherv", 2, "u8:heap:70001:out,f32:host:4099:out"),
    ("gatherv", 4, "f64:heap:4099:out,i64:heap:257:out"),
    ("scatterv", 2, "i64:heap:4099:out,u8:host:1501:out"),
    ("scatterv", 4, "f32:heap:70001:out,f64:heap:5:out"),
    ("allgatherv", 2, "f32:heap:4099:out,u8:host:257:out"),
    ("allgatherv", 4, "i64:heap:70001:out,f32:heap:3:out"),
    ("alltoallv", 2, "u8:heap:4099:out,f64:host:257:out"),
    ("alltoallv", 4, "f32:heap:70001:out,i64:heap:5:out"),
    ("barrier", 2, "f32:heap:0:out,f32:heap:0:out,f32:heap:0:out"),
    ("barrier", 4, "f32:heap:0:out"),
]


@pytest.mark.parametrize("family,n,variants", FAMILY_CASES, ids=["%s-n%d" % (f, n) for f, n, _ in FAMILY_CASES])
def test_collectives_on_both_sides_of_the_epoch_wrap(family, n, variants):
    """Each variant runs at the last launches before the scrub whose end value is 0 and at the first
    launches after it (start 1), every result against the oracle, the epoch checked after every call."""
    world(n, "wrap_family", "--family", family, "--variants", variants)


def test_oneshot_with_every_mid_barrier_value_at_the_wrap():
    """One CTA and a message whose plan has rounds == kMaxMids: the in-place one-shot uses every mid
    value of its stride, up to 2^32 - 4097 before the wrap and from 2 after it.  The count is chosen
    by oneshot_plan's rule (b200mpi.cu), restated here: with more rounds the library would fall back to
    two-shot and the worker's algorithm check would fail; with fewer, this assertion must change too."""
    count, blocks, threads, max_mids = 2095103, 1, 512, STRIDE - 2
    assert -(-count // (blocks * threads)) + 2 == max_mids  # plain (not shuffle) one-shot: 2 ranks, > 4096 vectors
    world(2, "wrap_family", "--family", "oneshot", "--variants", "f32:heap:%d:in" % count, "--max-blocks", str(blocks))


@pytest.mark.parametrize("family,n", [("ring", 2), ("ring", 4), ("allgather_ring", 3)])
def test_ring_kernels_across_the_ring_counter_wrap(family, n):
    """Ring step counters count epoch * 8 and wrap when the epoch passes 2^29: ring kernels on both
    sides of that launch."""
    variants = "f32:heap:65537:in,i64:heap:4099:out" if family == "ring" else "u8:heap:70001:out,f64:heap:257:out"
    world(n, "wrap_family", "--family", family, "--variants", variants, "--boundary", str(RING_WRAP), boundary=RING_WRAP)


@pytest.mark.parametrize("variant", ["f32:pageable:81923:out", "i64:pinned:40961:in"])
def test_pipelined_host_slices_straddle_the_wrap(variant):
    world(2, "wrap_hostpipe", "--variants", variant)


@pytest.mark.parametrize("what", ["count", "alltoallv"])
@pytest.mark.parametrize("n", [2, 4])
def test_mismatch_whose_resync_crosses_the_wrap(n, what):
    world(n, "wrap_mismatch", "--family", what)


LL_ENV = {"B200MPI_LL_SEQ_START": str((1 << 32) - 5)}


@pytest.mark.parametrize("n,kind", [(2, "heap"), (2, "host"), (4, "heap")])
def test_ll_allreduce_at_sequence_zero(n, kind):
    """The call that would get sequence 0 carries the largest message so far, with rank 1 late: the
    lanes beyond the earlier messages still hold the zeros of Init.  Bit-exact on every rank."""
    res = world(n, "ll_wrap", "--family", "plain", "--kinds", kind, env=LL_ENV)
    assert all(0 < r["ll_seq"] < 16 for r in res)


@pytest.mark.parametrize("kind", ["heap", "host"])
def test_ll_allreduce_after_a_resync_across_the_wrap(kind):
    world(2, "ll_wrap", "--family", "resync", "--kinds", kind, env=LL_ENV)


def test_ranks_with_different_epoch_starts_fail_init():
    starts = {0: start_below(EPOCH_WRAP), 1: start_below(EPOCH_WRAP, 13)}
    res = run_world(2, "smoke", timeout=300, env=dict(ENV), per_rank_env=lambda r: {"B200MPI_EPOCH_START": starts[r]})
    for r in res:
        assert not r.get("ok"), r
        assert "(b200mpi error %d)" % L.ERR_ARG in (r.get("error") or "") and "disagree" in r["error"], r.get("error")


def crossed(results, start, boundary, key="epoch"):
    """Every rank ended past `boundary` (mod 2^32) after starting at `start`."""
    for r in results:
        moved = (r[key] - start) % (1 << 32)
        assert moved > (boundary - start) % (1 << 32), "rank %d: %s went %d -> %d, short of %d" % (r["rank"], key, start, r[key], boundary)


@pytest.mark.parametrize("boundary", [1 << 31, 1 << 32], ids=["2^31", "2^32"])
def test_existing_scenarios_across_the_sign_half_and_the_wrap(boundary):
    """The collectives and newcolls scenarios, which make hundreds of launches, started 40 launches below
    2^31 (where a zeroed flag word would look ahead) and below 2^32; each must end past the boundary."""
    start = boundary - 40 * STRIDE + 1
    env = dict(ENV, B200MPI_EPOCH_START=str(start))
    for args in (["collectives", "--sizes", "1,257,65537", "--kinds", "heap,host", "--dtypes", "f32,i64"],
                 ["newcolls", "--sizes", "1,257,4099", "--kinds", "heap", "--dtypes", "f64,i64"]):
        res = run_world(2, "across", args=["--family"] + args[:1] + args[1:], timeout=900, env=env)
        assert_world_ok(res)
        crossed(res, start, boundary)


def test_switch_paths_across_the_wrap_on_real_nvlink():
    """NVLS, hybrid and LL with the wrap inside the run.  They cannot run when ranks share one GPU:
    shown as SKIPPED there, never as passed."""
    have = need_gpus(2, "multimem (NVLS) kernels")
    n = 8 if have >= 8 else 4 if have >= 4 else 2
    start, ll_start = (1 << 32) - 40 * STRIDE + 1, (1 << 32) - 20
    env = dict(ENV, B200MPI_EPOCH_START=str(start), B200MPI_LL_SEQ_START=str(ll_start), B200MPI_HEAP_BYTES=str(512 << 20))
    res = run_world(n, "across", args=["--family", "collectives", "--algos", "nvls,hybrid,ll", "--sizes", "1,257,4096,40001", "--kinds", "heap"],
                    timeout=900, env=env)
    assert_world_ok(res)
    assert all(r["nvls"] for r in res), "multicast mapping was not set up on a multi-GPU box"
    assert_nothing_skipped(res)
    crossed(res, start, 1 << 32)
    crossed(res, ll_start, 1 << 32, key="ll_seq")
