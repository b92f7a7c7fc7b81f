"""GPU tests of Send, Isend, Wait and Receive (run on an H100: pytest -m gpu).  The rank processes run
_p2p_worker.py: every sender layout against every receiver layout of _p2p_plan.py, with guarded buffers
of every memory kind, each call checked byte for byte, for the heap it leaves and for the kernels each
side launched; truncation and dtype mismatches against every sender layout, blocked rings included;
self-sends; 16 outstanding Isends; a short heap; and every ordered pair at once from threads.
When the box has fewer GPUs than ranks, the ranks share device 0."""
import os

import pytest

import _p2p_plan as P
from _launch import assert_world_ok, run_world

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_p2p_worker.py")
ENV = {"B200MPI_WATCHDOG_S": "90"}


def world(n, parts, *args, env=None, timeout=1200):
    e = dict(ENV)
    if env:
        e.update(env)
    res = run_world(n, "p2p", args=["--parts", parts] + list(args), timeout=timeout, env=e, worker=WORKER)
    assert_world_ok(res)
    for r in res:
        print("rank %d: %d calls %s seconds %s" % (r["rank"], r["checked"], r["by_part"], r["seconds"]))
    return res


def reached(res):
    out = {}
    for r in res:
        for k, v in r["pairs"].items():
            out[tuple(k.split("|"))] = out.get(tuple(k.split("|")), 0) + v
    return out


def check_pairs(n, res, want):
    got = reached(res)
    print("world of %d: %d (sender, receiver) layout pairs reached: %s" % (n, len(got), dict(sorted(got.items()))))
    missing = set(want) - set(got)
    assert not missing, "planned layout pairs that never ran: %s" % sorted(missing)


def test_layout_matrix_world_of_2():
    """The whole matrix, both directions; truncation and mismatch against every sender layout; self-sends
    on both ranks; 16 outstanding Isends and the 17th refused."""
    res = world(2, "matrix,errors,self,depth")
    check_pairs(2, res, {c.pair() for _, _, c in P.matrix()})


def test_layout_matrix_world_of_3():
    """Every third matrix case from rank 0 to rank 2, which is not its neighbour; self-sends on every rank."""
    res = world(3, "matrix,self")
    check_pairs(3, res, {c.pair() for _, _, c in P.matrix(3, 0, 2, stride=3)})


def test_large_messages_at_the_default_chunk():
    """160 MiB host and heap Sends at the default 32 MiB chunk (rings that wrap, a direct post pulled in
    32 MiB units), and rings whose chunks are larger than the receiver's stage_chunk."""
    res = world(2, "big", env={"B200MPI_HEAP_BYTES": str(512 << 20)})
    check_pairs(2, res, {c.pair() for c in P.big_cases()})


@pytest.mark.parametrize("case", ["a", "b", "c"])
def test_heap_pressure(case):
    """(a) 96 MiB heap and pageable messages into host memory with 8 MiB of heap free; (b) a receive with
    no room to stage fails with B200MPI_ERR_NOMEM and leaves the message posted for a retry; (c) an Isend
    larger than the free heap fails and releases its slot and tag."""
    world(2, "pressure_" + case, env={"B200MPI_HEAP_BYTES": str(256 << 20)}, timeout=600)


@pytest.mark.parametrize("n", [3, 4])
def test_every_pair_at_once(n):
    """Every ordered pair, self included, 3 messages each, from threads; 2n host-slice sends of at most
    4 MiB per rank in flight, more than the 4 mapped bounces."""
    res = world(n, "concurrent", "--tags", "3")
    assert all(r["host_sends_in_flight"] >= 6 for r in res), [r["host_sends_in_flight"] for r in res]


def test_every_pair_at_once_world_of_8():
    """As above with 2 host-slice messages per ordered pair, at most 1 MiB each."""
    res = world(8, "concurrent", "--tags", "2")
    assert all(r["host_sends_in_flight"] >= 6 for r in res), [r["host_sends_in_flight"] for r in res]
