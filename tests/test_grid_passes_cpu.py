"""The pass planner of _passes_worker.py without a GPU: the grid rules it restates, pinned to the
lines of b200mpi.cu and kernels.cuh they come from; two hand-worked cases; and every count that
test_gpu_grid_passes.py runs reaching the passes it is planned for."""
import os
import re

import pytest

import _passes_worker as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLDS = [2, 3, 4, 6, 8]
CAPS = [1, 3]


def source(name):
    with open(os.path.join(ROOT, "mpi_b200", "csrc", name)) as f:
        return re.sub(r"\s+", " ", f.read())


# The lines of the library the planner restates.  When one of them changes, the planner must follow.
RULES_CU = [
    "int cap = g->max_blocks > 0 ? std::min(g->max_blocks, g->sm_count) : g->sm_count; return std::min(cap, kMaxBlocks);",
    "size_t per_block = (size_t)kThreads * unroll; size_t want = (units_per_rank + per_block - 1) / per_block; int cap = block_cap(); if (want < 1) want = 1;",
    "while (((size_t)2 << sh) <= per) ++sh;",
    "while (((size_t)32 << cap) <= g->own_block_bytes) ++cap;",
    "if (n == 2) return f(ic<2>{}, ic<sizeof(T) == 4 ? 8 : 4>{}); if (n == 4) return f(ic<4>{}, ic<4>{}); if (n == 8) return f(ic<8>{}, ic<2>{}); return f(ic<0>{}, ic<1>{});",
    "const uint32_t sh = own_shift(nvec, n, algo == B200MPI_ALGO_TWOSHOT_SMEM ? 8 : 0);",
    "grid_for(per, unroll), kThreads, 0, s, so, ro, count, sh, only_dst);",
    "\"allreduce_ring_kernel\", sig, grid_for(per, 4)",
    "const size_t tiles = (per * 16 + kSmemChunk - 1) / kSmemChunk; const int blocks = (int)std::max<size_t>(1, std::min<size_t>(tiles, (size_t)block_cap()));",
    "p.shfl = (n == 2 || n == 4 || n == 8) && nvec <= 4096; p.blocks = p.shfl ? grid_for(nvec * n, 1) : grid_for(nvec, 1);",
    "\"reduce_scatter_kernel\", sig, grid_for(nvec, 2)",
    "\"scan_kernel\", sig, grid_for(per, unroll)",
    "const int blocks = grid_for(mode ? nvec / (size_t)(n - 1) + 1 : nvec, 4);",
    "const int blocks = grid_for(bytes / 16 + 1, 4);",
    "return grid_for(largest / 16 + 1, unroll);",
    "constexpr int U = sizeof(T) == 4 ? 8 : 4;",
    "\"reduce_scatterv_kernel\", sig, vtable_grid(vt, U)",
    "const int blocks = block_cap();",
    "const int blocks = (int)std::max<size_t>(1, std::min<size_t>((ncell + 255) / 256, 128));",
    "constexpr size_t kPerBlock = 256 * 16 * 16;",
    "const size_t cap = g->max_blocks > 0 ? (size_t)g->max_blocks : (size_t)g->sm_count;",
    "size_t p2p_vec = (size_t)((double)nvec * g->hybrid_p2p_permille / 1000.0); const size_t gran = (size_t)n << 8;",
    "int u = g->nvls_unroll == 4 ? 4 : 2; const int nb_nvls = nvls_blocks((split + n - 1) / n, u);",
    "int nb_p2p = g->hybrid_p2p_blocks > 0 ? g->hybrid_p2p_blocks : block_cap() - nb_nvls; nb_p2p = std::max(1, std::min(nb_p2p, block_cap() - nb_nvls)); if (nb_nvls + nb_p2p > block_cap()) return launch_allreduce_nvls_t<T, Op>(sig, so, ro, count, -1, s);",
    "if (g->max_blocks == 0 && blocks > g->nvls_max_blocks) blocks = g->nvls_max_blocks;",
]
RULES_CUH = [
    "constexpr int kMaxBlocks = 528;",
    "constexpr int kThreads = 512;",
    "constexpr size_t kLLRegionCells = 2 * 8 * 32768;",
    "constexpr int kSmemChunk = 4096;",
    "constexpr int kSmemStages = 4;",
    "const size_t nblk = (nvec_ + ((size_t)1 << shift_) - 1) >> shift_; const size_t mine = nblk > (size_t)rank_ ? (nblk - rank_ + n_ - 1) / n_ : 0;",
    "for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) { if (own.global(t * kTileVecs) >= nvec) continue;",
    "const size_t step = (size_t)nb * blockDim.x * UNROLL;",
    "copy_bytes_kernel(unsigned char* __restrict__ dst, const unsigned char* __restrict__ src, size_t bytes) {",
]


@pytest.mark.parametrize("name,lines", [("b200mpi.cu", RULES_CU), ("kernels.cuh", RULES_CUH)])
def test_the_restated_rules_are_the_librarys(name, lines):
    text = source(name)
    missing = [ln for ln in lines if ln not in text]
    assert not missing, "%s no longer holds these grid rules; update _passes_worker.py's planner to follow: %s" % (name, missing)


def test_twoshot_world_of_4_cap_1_hand_worked():
    """f32, default knobs (UNROLL 4, own_block_bytes 1 MiB), nvec = 24576: per = 6144, so the shift
    is 12, nblk = 6 and the ranks hold 8192 / 8192 / 4096 / 4096 slots: 4, 4, 2 and 2 passes of 2048."""
    R = P.Rules(4, 1)
    count = 24576 * 4
    nvec, sh, per = P._owner(R, count, 4)
    assert (nvec, sh, per) == (24576, 12, 6144)
    assert R.tiling(4) == (4, 4)
    assert [R.owner_slots(nvec, sh, r) for r in range(4)] == [8192, 8192, 4096, 4096]
    assert [P.loop_passes(R.owned(nvec, sh, r), 1, 2048) for r in range(4)] == [[4], [4], [2], [2]]
    assert P.passes(R, "twoshot", count, 4) == [4]


def test_smem_world_of_4_cap_1_hand_worked():
    """f32, nvec = 9316: the shift is 11 (8 tiles per block).  Rank 0 owns blocks 0 and 4 and takes 13
    tiles, the 13th 100 vectors long, and skips 3; rank 3 takes 8."""
    R = P.Rules(4, 1)
    grid, ranks = P.smem_tiles(R, 9316 * 4, 4)
    assert grid == 1
    assert ranks[0]["shift"] == 11
    assert ranks[0]["ctas"] == [(13, 3)] and ranks[0]["last_tile"] == 100
    assert ranks[3]["ctas"] == [(8, 0)]


def test_one_shot_forms_and_rounds():
    for n in WORLDS:
        for cap in CAPS:
            R = P.Rules(n, cap)
            for es in (4, 8):
                for c in P.plan(R, "oneshot", es).values():
                    shfl, blocks, rounds = R.oneshot_plan(c, es)
                    assert not shfl and blocks == cap and rounds <= P.MAX_MIDS
                if n in (2, 4, 8):
                    for c in P.plan(R, "oneshot_shfl", es).values():
                        shfl, blocks, rounds = R.oneshot_plan(c, es)
                        assert shfl and blocks == cap and rounds <= P.MAX_MIDS


KERNELS = ["oneshot", "oneshot_shfl", "twoshot", "reduce", "ring", "reduce_scatter", "scan", "exscan",
           "bcast", "bcast2", "allgather", "allgather_ring", "alltoall", "copy"]


@pytest.mark.parametrize("n", WORLDS)
@pytest.mark.parametrize("cap", CAPS)
def test_every_planned_count_reaches_its_passes(n, cap):
    """exact: every CTA of the busiest rank makes 3 passes (the rank-order one-shot in worlds of 2, 4
    and 8 more, to stay above the shuffle form's 4096 vectors).  plus1: CTA 0 one more.  partial: the
    last CTA's last pass leaves UNROLL slots (or, at UNROLL 1, threads) empty.  A count % EPV tail on
    every reduction count."""
    R = P.Rules(n, cap)
    for kernel in KERNELS:
        if kernel == "oneshot_shfl" and n not in (2, 4, 8):
            continue
        for es in ((4, 8) if kernel in P.LOOPS and kernel not in ("bcast", "bcast2", "allgather", "allgather_ring", "alltoall", "copy") else (1, 4, 8)):
            counts = P.plan(R, kernel, es)
            units, grid, per_cta, lane = P.LOOPS[kernel](R, counts["exact"], es)
            assert grid == cap, (kernel, es, grid)
            exact = P.passes(R, kernel, counts["exact"], es)
            q = exact[0]
            assert q >= 3 and exact == [q] * grid, (kernel, es, exact)
            assert P.passes(R, kernel, counts["plus1"], es) == [q + 1] + [q] * (grid - 1), (kernel, es)
            partial = P.passes(R, kernel, counts["partial"], es)
            assert partial == [q] * grid, (kernel, es, partial)
            units, _, _, _ = P.LOOPS[kernel](R, counts["partial"], es)
            last = units - (q - 1) * grid * per_cta - (grid - 1) * per_cta
            assert last == per_cta - lane + 7, (kernel, es, last)  # the last slot holds 7 threads' units
            if kernel in ("oneshot", "oneshot_shfl", "twoshot", "reduce", "ring", "reduce_scatter", "scan", "exscan"):
                assert all(c % (16 // es) for c in counts.values()), (kernel, es, counts)
            if "tail" in counts:
                assert min(P.passes(R, kernel, counts["tail"], es)) >= q


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("cap", CAPS)
def test_smem_plans_wrap_the_stage_ring(n, cap):
    """Every CTA of rank 0 takes 4, 9 (= 2 * kSmemStages + 1: the mbarrier parity has come back) and
    12 tiles, the last 100 vectors long; from 9 tiles on its second block is partial, so tiles are
    skipped, and every block is bigger than one tile."""
    R = P.Rules(n, cap)
    for es in (4, 8):
        for name, c in P.smem_plan(R, es).items():
            t = int(name[len("tiles"):])
            grid, ranks = P.smem_tiles(R, c, es)
            assert grid == cap
            assert [x[0] for x in ranks[0]["ctas"]] == [t] * cap, (name, ranks[0])
            assert ranks[0]["last_tile"] == 100 and ranks[0]["shift"] > 8
            assert max(min(x[0] for x in r["ctas"]) for r in ranks) == t
            if t >= 9:
                assert sum(x[1] for x in ranks[0]["ctas"]) > 0


@pytest.mark.parametrize("n", WORLDS)
@pytest.mark.parametrize("cap", CAPS)
def test_table_plans_and_ll(n, cap):
    """The v-collectives' and Alltoallv's largest block and ReduceScatterv's make >= 3 passes per CTA;
    LL (whose grid ignores the cap) goes past 32768 cells where the world's lanes allow it."""
    R = P.Rules(n, cap)
    counts, skew = P.v_table(R, 1)
    assert P.passes(R, "v", counts, 1)[-1] >= 3
    assert P.passes(R, "alltoallv", skew, 1) == [3] * cap
    for es in (4, 8):
        rsv = P.rsv_table(R, es)
        assert rsv[0] % (16 // es) and P.passes(R, "rsv", rsv, es) == [3] * cap
        ll = P.plan(R, "ll", es)
        for c in ll.values():
            cells = c * es // 8
            assert cells <= P.ll_cells(n)
        if n <= 4:
            assert P.passes(R, "ll", ll["plus1"], es) == [2] + [1] * 127
            assert P.passes(R, "ll", ll["partial"], es) == [2] * 128


@pytest.mark.parametrize("n", [2, 4, 8])
def test_hybrid_needs_a_cta_for_each_part(n):
    """A hybrid request runs the NVLS kernel under cap 1 at any count; at hybrid_plan's count under
    cap 3 the fused kernel runs with 2 NVLS CTAs and 1 P2P CTA, whose two-shot body makes 4 passes or
    more."""
    for es in (4, 8):
        for unroll in (2, 4):
            for count in [1, 257, 4097, 40001, 1048577, P.hybrid_plan(P.Rules(n, 3), es, unroll)]:
                assert P.hybrid_grid(P.Rules(n, 1), count, es, P.HYBRID_PERMILLE, unroll) is None
            count = P.hybrid_plan(P.Rules(n, 3), es, unroll)
            nb_nvls, nb_p2p, p2p = P.hybrid_grid(P.Rules(n, 3), count, es, P.HYBRID_PERMILLE, unroll)
            assert (nb_nvls, nb_p2p) == (2, 1)
            _, up = {2: (2, 4), 4: (4, 4), 8: (8, 2)}[n]
            assert p2p // n // (512 * up) >= 4
