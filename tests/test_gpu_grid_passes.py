"""GPU tests of every collective kernel past its first grid pass (run on an H100: pytest -m gpu).  The
rank processes run _passes_worker.py: under b200mpi_set_max_blocks(1) and (3) each kernel runs every
count the planner chose -- 3 passes per CTA of its busiest rank exactly, one vector more, and a
partial last pass; the TMA two-shot 4, 9 and 12 tiles per CTA -- in every dtype on 16-byte aligned
heap buffers, where its vector loop runs, then once per unaligned layout and once on host views, with
the footprint checks of test_gpu_footprint.py.  Then ranks whose grids differ must refuse every
signed call.
When the box has fewer GPUs than ranks, the ranks share device 0."""
import os

import pytest

from _launch import assert_world_ok, run_world
from test_gpu_worlds import assert_nothing_skipped, need_gpus

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_passes_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}
# the kernels the full set runs at >= 3 passes per CTA of the busiest rank (LL, whose grid ignores
# the cap, at its planned counts past 32768 cells)
FULL = {"oneshot", "twoshot", "ring", "reduce", "reduce_scatter", "scan", "exscan", "rsv", "bcast", "bcast2",
        "allgather", "allgather_ring", "alltoall", "v", "alltoallv", "copy"}


def world(n, scenario, *args, env=None, timeout=1200):
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, scenario, args=list(args), timeout=timeout, env=e, worker=WORKER)
    assert_world_ok(res)
    return res


def check_passes(n, res, kernels):
    """Every kernel ran every plan in every dtype on aligned heap buffers, plus its unaligned and host
    calls; each reached its planned passes (the TMA form its 4, 9 and 12 tiles per CTA)."""
    r0 = res[0]
    print("world of %d: %d calls checked per rank %s" % (n, r0["checked"], r0["by_part"]))
    for cap, got in sorted(r0["caps"].items()):
        print("  cap %s: fewest passes per CTA on the busiest rank %s, TMA tiles per CTA %s, seconds %s" % (
            cap, dict(sorted(got["min_passes"].items())), got["smem_tiles"], got["seconds"]))
        want = kernels | ({"oneshot_shfl", "smem"} if n in (2, 4, 8) else set())
        want = want if cap == "1" else want - {"ll"}  # LL runs once: its grid ignores the cap
        ran, planned = got["ran_aligned"], got["planned"]
        assert want <= set(planned), "cap %s: kernels not run: %s" % (cap, sorted(want - set(planned)))
        for k in want:
            assert ran.get(k) == planned[k], "cap %s: %s ran aligned %s of %s" % (cap, k, ran.get(k), planned[k])
            if k not in ("v", "alltoallv", "copy"):
                kinds = got["extra"].get(k, [])
                assert sum(1 for x in kinds if x.split("/")[-1] in ("symmetric", "mixed", "split")) == 3, (cap, k, kinds)
                assert any(x.endswith("/host") for x in kinds), (cap, k, kinds)
        low = {k: v for k, v in got["min_passes"].items() if k not in ("ll", "smem") and v < 3}
        assert not low, "cap %s: kernels below their planned passes: %s" % (cap, low)
        if n in (2, 4, 8):
            assert got["smem_tiles"] == {"tiles4": 4, "tiles9": 9, "tiles12": 12}, got["smem_tiles"]


@pytest.mark.parametrize("n", [2, 3, 4, 6])
def test_every_kernel_past_its_first_grid_pass(n):
    res = world(n, "passes", "--set", "full")
    check_passes(n, res, FULL | {"ll"} if n <= 4 else FULL)


def test_every_kernel_past_its_first_grid_pass_world_of_8():
    """The reductions, byte-moving collectives and Send / Receive (no v-collectives, no LL)."""
    res = world(8, "passes", "--set", "reduced")
    check_passes(8, res, FULL - {"v", "alltoallv"})


@pytest.mark.parametrize("n", [2, 4])
def test_ranks_with_different_grids_refuse_the_call(n):
    """Rank 0 at cap 1, the others at 3 (rank 3 of the world of 4 uncapped): two-shot, TMA two-shot and
    ring Allreduce, Bcast, ReduceScatter and Alltoallv end as B200MPI_ERR_PEER on every rank with
    nothing written, heap and staged host alike, the epoch advanced alike; the LL Allreduce succeeds."""
    res = world(n, "grids")
    r0 = res[0]
    print("world of %d: caps %s, refused %d calls per rank, %d LL calls matched, epoch steps %s" % (
        n, [r["cap"] for r in res], len(r0["refused"]), r0["ll_under_different_caps"], r0["epoch_steps"]))
    assert len({r["cap"] for r in res}) > 1
    steps = [r["epoch_steps"] for r in res]
    assert all(s == steps[0] for s in steps), "the epoch advanced differently on the ranks: %s" % steps
    assert all(r["refused"] and len(r["refused"]) == len(r0["refused"]) for r in res)
    assert r0["ll_under_different_caps"] >= 2


def test_switch_paths_past_their_first_grid_pass():
    """The switch paths of test_gpu_footprint.py (NVLS and hybrid Allreduce, NVLS Reduce, ReduceScatter
    and both NVLS Bcasts) under caps 1 and 3; nvls_blocks ignores nvls_max_blocks once a cap is set.
    A hybrid request needs a CTA for each part: under cap 1 it runs the NVLS kernel, and under cap 3
    the fused kernel runs only where its NVLS part needs 2 CTAs or fewer.  So the hybrid Allreduce also
    runs at hybrid_plan's count, where the fused kernel gets 2 NVLS CTAs and 1 P2P CTA under cap 3.
    They cannot run when ranks share one GPU: shown as SKIPPED there, never as passed."""
    have = need_gpus(2, "multimem (NVLS) kernels")
    n = 8 if have >= 8 else 4 if have >= 4 else 2
    res = world(n, "passes", "--set", "nvls", env={"B200MPI_HEAP_BYTES": str(512 << 20)})
    assert all(r["nvls"] for r in res), "multicast mapping was not set up on a multi-GPU box"
    assert_nothing_skipped(res)
    hybrid = {cap: got["extra"]["hybrid"] for cap, got in res[0]["caps"].items()}
    print("world of %d: hybrid calls %s" % (n, hybrid))
    assert all("NVLS kernel" in x for x in hybrid["1"]) and all("fused kernel" in x for x in hybrid["3"]), hybrid
