"""The point-to-point planner of _p2p_plan.py without a GPU: the rules it restates, pinned to the lines
of the library they come from; hand-worked cases; and every count it plans reaching the layouts it is
planned for."""
import itertools
import os
import re

import pytest

import _p2p_plan as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KB, MB = P.KB, P.MB


def source(name):
    with open(os.path.join(ROOT, "mpi_b200", "csrc", name)) as f:
        return re.sub(r"\s+", " ", f.read())


# The lines of the library the planner restates.  When one of them changes, the planner must follow.
RULES_CU = [
    "constexpr int kSlotsPerPair = 16;",
    "constexpr int kMsgRegions = 4;",
    "static constexpr int kP2PBounces = 4;",
    "static constexpr size_t kP2PBounceBytes = 4u << 20;",
    "size_t stage_chunk = 32u << 20;",
    "if (memkind == B200MPI_HOST) return std::min(g->stage_chunk, std::max<size_t>(64u << 10, (bytes / 4 + 4095) / 4096 * 4096)); return g->stage_chunk;",
    # do_send
    "const bool direct = bytes == 0 || (wait_ack && memkind == B200MPI_DEVICE && g->heap.contains(buf, bytes, off));",
    "Ctx::P2PBounce* bounce = !direct && memkind == B200MPI_HOST && g->p2p_fast && bytes <= Ctx::kP2PBounceBytes ? acquire_bounce() : nullptr;",
    "const size_t chunk = direct || bounce || !wait_ack ? bytes : std::min(bytes, p2p_chunk(bytes, memkind));",
    "const size_t nchunks = direct ? 0 : (bytes + chunk - 1) / chunk;",
    "const size_t nreg = std::min<size_t>(std::max<size_t>(nchunks, 1), kMsgRegions);",
    "if (g->heap.alloc(chunk * nreg, ps.stage))",
    "memcpy(bounce->host, from, len); rc = copy_and_wait(bounce, to, bounce->dev, len, s);",
    "if (memkind == B200MPI_HOST) e = cudaMemcpyAsync(to, from, len, cudaMemcpyHostToDevice, s); else rc = launch_copy(to, from, len, s);",
    # copy_and_wait and launch_copy: two launches through a bounce, none for an empty copy
    "int rc = launch_copy(dst, src, bytes, s); if (rc) return rc; const uint32_t seq = ++b->seq; flag_kernel<<<1, 1, 0, s>>>",
    "static int launch_copy(void* dst, const void* src, size_t bytes, cudaStream_t s) { if (bytes == 0) return 0;",
    # do_recv
    "if (rc == 0 && bytes && memkind == B200MPI_HOST && g->p2p_fast && chunk * nreg >= bytes && bytes <= Ctx::kP2PBounceBytes) bounce = acquire_bounce();",
    "const size_t unit = bounce ? bytes : memkind == B200MPI_HOST ? std::min(chunk, g->stage_chunk) : chunk;",
    "const bool staged = rc == 0 && bytes && !bounce && memkind == B200MPI_HOST;",
    "len = bounce ? bytes : std::min({unit, chunk - lo % chunk, bytes - lo});",
    "const char* from = peer + slot->region_off[lo / chunk % nreg] + lo % chunk;",
    "rc = copy_and_wait(bounce, bounce->dev, from, len, s);",
    "rc = launch_copy(memkind == B200MPI_DEVICE ? (char*)buf + lo : mine + stage, from, len, s);",
]
RULES_HEAP = ["const size_t a = 512;"]


@pytest.mark.parametrize("name,lines", [("b200mpi.cu", RULES_CU), ("heap.cpp", RULES_HEAP)])
def test_the_restated_rules_are_the_librarys(name, lines):
    text = source(name)
    missing = [ln for ln in lines if ln not in text]
    assert not missing, "%s no longer holds these point-to-point rules; update _p2p_plan.py to follow: %s" % (name, missing)


def test_pageable_ring_into_pinned_hand_worked():
    """1 MiB + 4 bytes from pageable memory with p2p_fast off at stage_chunk 256 KiB: a quarter is 262145 bytes, 266240
    rounded up to 4 KiB, so the chunk is capped at 256 KiB; 5 chunks through 4 regions (the fifth reuses
    region 0), filled by cudaMemcpyAsync.  Four regions hold 1 MiB, less than the message, so a pinned
    receiver does not bounce: 5 units of 256 KiB, the last 4 bytes long."""
    sp = P.plan_send(MB + 4, host=True, in_heap=False, isend=False, fast=False, stage_chunk=256 * KB)
    assert sp == P.SendPlan("ring/memcpy", 256 * KB, 5, 4, MB, 0)
    rp = P.plan_recv(sp, MB + 4, host=True, fast=True, stage_chunk=256 * KB)
    assert rp == P.RecvPlan("staged", 256 * KB, 5, 256 * KB, 5)
    assert P.pull_units(MB + 4, sp.chunk, rp.unit)[-1] == (MB, 4)


def test_heap_send_into_pageable_stages_one_chunk_hand_worked():
    """A 160 MiB + 4 byte heap Send is posted direct, as one chunk of the whole message.  A pageable
    receiver at the default stage_chunk pulls it in 6 units of at most 32 MiB and stages 32 MiB, as
    much as the same message sent from pageable memory costs it (a ring of 32 MiB chunks)."""
    nbytes = 160 * MB + 4
    sp = P.plan_send(nbytes, host=False, in_heap=True, isend=False, fast=True, stage_chunk=P.STAGE_CHUNK)
    assert sp == P.SendPlan("direct", nbytes, 0, 1, 0, 0)
    rp = P.plan_recv(sp, nbytes, host=True, fast=True, stage_chunk=P.STAGE_CHUNK)
    assert rp == P.RecvPlan("staged-split", 32 * MB, 6, 32 * MB, 6)
    ring = P.plan_send(nbytes, host=True, in_heap=False, isend=False, fast=True, stage_chunk=P.STAGE_CHUNK)
    assert (ring.layout, ring.chunk, ring.nchunks, ring.nreg, ring.stage) == ("ring/memcpy", 32 * MB, 6, 4, 128 * MB)
    assert P.plan_recv(ring, nbytes, host=True, fast=True, stage_chunk=P.STAGE_CHUNK).stage == rp.stage


def test_isend_and_bounce_hand_worked():
    """A 3 MiB torch Isend is one staged chunk, one kernel; a pinned receiver with p2p_fast bounces it
    (2 launches).  A 100 KiB pageable Send with p2p_fast bounces too (2 launches, no ring), and with
    p2p_fast off is a 2-chunk ring of 64 KiB."""
    sp = P.plan_send(3 * MB, host=False, in_heap=False, isend=True, fast=False, stage_chunk=256 * KB)
    assert sp == P.SendPlan("whole/kernel", 3 * MB, 1, 1, 3 * MB, 1)
    assert P.plan_recv(sp, 3 * MB, host=True, fast=True, stage_chunk=256 * KB) == P.RecvPlan("bounce", 3 * MB, 1, 0, 2)
    assert P.plan_recv(sp, 3 * MB, host=False, fast=True, stage_chunk=256 * KB) == P.RecvPlan("device", 3 * MB, 1, 0, 1)
    assert P.plan_send(100 * KB, True, False, False, True, 256 * KB) == P.SendPlan("whole/bounce", 100 * KB, 1, 1, 100 * KB, 2)
    assert P.plan_send(100 * KB, True, False, False, False, 256 * KB) == P.SendPlan("ring/memcpy", 64 * KB, 2, 2, 128 * KB, 0)
    # every bounce taken: the same message is a ring
    assert P.plan_send(100 * KB, True, False, False, True, 256 * KB, bounce_free=False).layout == "ring/memcpy"


def test_units_never_cross_a_chunk_end():
    for nbytes, chunk, unit in ((10 * MB + 3, 3 * MB, MB), (7 * MB, 7 * MB, 2 * MB), (5, 5, 5), (MB + 1, 300 * KB, 256 * KB)):
        units = P.pull_units(nbytes, chunk, unit)
        assert sum(n for _, n in units) == nbytes and units[0][0] == 0
        assert all(a + n == b for (a, n), (b, _) in zip(units, units[1:]))
        assert all(0 < n <= unit and lo // chunk == (lo + n - 1) // chunk for lo, n in units)


@pytest.mark.parametrize("dt", P.DTYPES)
def test_boundary_counts_sit_either_side_of_every_rule(dt):
    """For each boundary the count one element below and one above take different layouts or shapes."""
    es, sc = P.ESIZE[dt], 256 * KB
    counts = P.boundary_counts(dt, sc)
    assert counts[0] == 0
    b = P.boundaries(sc)

    def host_ring(c):
        return P.plan_send(c * es, True, False, False, False, sc)

    def dev_ring(c):
        return P.plan_send(c * es, False, False, False, False, sc)

    lo, hi = b["one host chunk"] // es - 1, b["one host chunk"] // es + 1
    assert (host_ring(lo).nchunks, host_ring(hi).nchunks) == (1, 2)
    lo, hi = b["quarter crosses 64 KiB"] // es - 1, b["quarter crosses 64 KiB"] // es + 1
    assert host_ring(lo).chunk == P.HOST_MIN_CHUNK < host_ring(hi).chunk
    lo, hi = b["one device chunk"] // es - 1, b["one device chunk"] // es + 1
    assert (dev_ring(lo).nchunks, dev_ring(hi).nchunks) == (1, 2)
    lo, hi = b["ring wraps"] // es - 1, b["ring wraps"] // es + 1
    for ring in (host_ring, dev_ring):
        assert (ring(lo).nchunks, ring(hi).nchunks) == (4, 5)
        assert P.plan_recv(ring(lo), lo * es, True, True, sc).layout == "bounce"
        assert P.plan_recv(ring(hi), hi * es, True, True, sc).layout == "staged"
    lo, hi = b["bounce"] // es - 1, b["bounce"] // es + 1
    assert P.plan_send(lo * es, True, False, True, True, sc).layout == "whole/bounce"
    assert P.plan_send(hi * es, True, False, True, True, sc).layout == "whole/memcpy"
    iso = P.plan_send(lo * es, False, False, True, True, sc), P.plan_send(hi * es, False, False, True, True, sc)
    assert P.plan_recv(iso[0], lo * es, True, True, sc).layout == "bounce"
    assert P.plan_recv(iso[1], hi * es, True, True, sc).layout == "staged-split"
    for c in counts:
        assert c == 0 or any(c in (x // es - 1, x // es + 1) for x in b.values())


def test_every_planned_pair_is_reached():
    """The matrix and the big cases reach every (sender, receiver) layout pair the library has: all of
    them, except an empty message in any layout but direct (an empty message is always direct); the
    matrix reaches each of its pairs at least 4 times."""
    want = set(itertools.product(P.SEND_LAYOUTS, P.RECV_LAYOUTS)) - {(s, "none") for s in P.SEND_LAYOUTS if s != "direct"}
    assert set(P.all_pairs()) == want
    cases = [c for _, _, c in P.matrix()]
    assert len(cases) == 7 * 7 * 2 * 4
    seen = {}
    for c in cases:
        seen[c.pair()] = seen.get(c.pair(), 0) + 1
    assert min(seen.values()) >= 4, seen
    # every storage pair, both calls and all four p2p_fast settings, every dtype and every count
    assert len({(c.send, c.recv, c.isend, c.send_fast, c.recv_fast) for c in cases}) == len(cases)
    assert {c.dtype for c in cases} == set(P.DTYPES)
    for dt in P.DTYPES:
        assert {c.count for c in cases if c.dtype == dt} == set(P.boundary_counts(dt))
    # the reduced matrix of the world of 3 still reaches most pairs
    assert len({c.pair() for _, _, c in P.matrix(3, 0, 2, stride=3)}) >= 16


def test_plans_are_self_consistent():
    """For every planned case: the regions hold at most 4 chunks and cover the message, the staging is
    the regions' size, and the launches follow the layout."""
    for _, _, c in P.matrix() + [(0, 1, x) for x in P.big_cases()]:
        sp, rp = c.plans()
        if sp.layout == "direct":
            assert sp.stage == 0 and sp.launches == 0
            continue
        assert 1 <= sp.nreg <= P.MSG_REGIONS and sp.chunk * sp.nchunks >= c.nbytes > sp.chunk * (sp.nchunks - 1)
        assert sp.stage == sp.chunk * sp.nreg
        assert sp.launches == {"bounce": 2, "memcpy": 0, "kernel": sp.nchunks}[sp.layout.split("/")[1]]
        if sp.layout.startswith("whole"):
            assert sp.nchunks == 1
        if rp.layout == "bounce":
            assert rp.launches == 2 and rp.stage == 0 and c.nbytes <= P.BOUNCE_BYTES
        elif rp.layout.startswith("staged"):
            assert rp.stage == rp.unit <= (c.recv_stage_chunk or c.stage_chunk) and rp.launches == rp.units

