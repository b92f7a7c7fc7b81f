"""One rank of a test world that runs every collective kernel past its first grid pass.
Usage as _worker.py: _passes_worker.py <passes|grids> --out FILE [--set full|reduced] -mpi-* flags.

Every kernel is a grid-stride loop: CTA b starts at b units and steps by the whole grid.  The host
caps the grid at the SM count, so a CTA loops only when a rank's share exceeds 132 CTAs' worth;
b200mpi_set_max_blocks lowers that cap for every launch.  The first half of this file restates the
grid rules of b200mpi.cu in plain Python (no GPU, no library): for a world of n ranks and a cap it
gives each kernel's grid and the passes every CTA of the busiest rank makes, and chooses counts
that reach a stated number of passes.  test_grid_passes_cpu.py pins it against hand-worked cases.

Scenario 'passes' runs, under caps 1 and 3, the calls of _footprint_worker.py (and the Scan and
ReduceScatterv footprints) at those counts, so every result is guarded and bit-exact in the order
of the kernel that ran.  Scenario 'grids' has rank 0 launch a smaller grid than the others: every
signed kernel must refuse the call on every rank with nothing written."""
import argparse
import ctypes
import os
import sys
import time

import numpy as np

# ---- the pass planner: b200mpi.cu's grid rules, pure Python ----------------------------------
THREADS = 512          # kThreads
SM_COUNT = 132         # H100 SXM
MAX_BLOCKS = 528       # kMaxBlocks
TILE_VECS = 4096 // 16  # kSmemChunk / 16: vectors per TMA tile
SMEM_STAGES = 4        # kSmemStages: the mbarrier parity repeats every 2 * 4 tiles
MAX_MIDS = 4096 - 2    # kMaxMids
LL_THREADS, LL_CTAS = 256, 128
LL_REGION_CELLS = 2 * 8 * 32768
COPY_THREADS, COPY_UNROLL = 256, 16  # launch_copy: copy_bytes_kernel<16, 256>


def cdiv(a, b):
    return -(-a // b)


def ll_cells(n):
    return LL_REGION_CELLS // (2 * max(n, 1))


class Rules:
    """The host's grid rules for a world of n ranks with b200mpi_set_max_blocks(cap) (0: no cap)."""

    def __init__(self, n, cap, sm_count=SM_COUNT, own_block_bytes=1 << 20, twoshot_unroll=True):
        self.n, self.cap, self.sm_count = n, cap, sm_count
        self.own_block_bytes, self.twoshot_unroll = own_block_bytes, twoshot_unroll

    def block_cap(self):
        c = min(self.cap, self.sm_count) if self.cap > 0 else self.sm_count
        return min(c, MAX_BLOCKS)

    def grid_for(self, units, unroll):
        return int(min(max(cdiv(units, THREADS * unroll), 1), self.block_cap()))

    def own_shift(self, nvec, min_shift=0):
        per = max(cdiv(nvec, self.n), 1)
        sh = per.bit_length() - 1
        cap = (self.own_block_bytes // 16).bit_length() - 1
        return max(min(sh, cap), min_shift)

    def tiling(self, es):
        """(NR, UNROLL) of the owner-computes kernels: with_owner_tiling, or the twoshot_unroll=0 table."""
        n = self.n
        if not self.twoshot_unroll:
            return {2: (2, 4), 4: (4, 2), 8: (8, 1)}.get(n, (0, 1))
        return {2: (2, 8 if es == 4 else 4), 4: (4, 4), 8: (8, 2)}.get(n, (0, 1))

    def owner_slots(self, nvec, shift, r):
        """Owner(nvec, shift, n, r).slots: this rank's blocks << shift (the last may be partial)."""
        nblk = cdiv(nvec, 1 << shift)
        mine = cdiv(nblk - r, self.n) if nblk > r else 0
        return mine << shift

    def owned(self, nvec, shift, r):
        """Vectors below nvec among rank r's slots: a prefix of them, since only the last block of
        the message is partial and it is its owner's last block."""
        b = 1 << shift
        return sum(min(b, max(0, nvec - (((q * self.n + r) << shift)))) for q in range(self.owner_slots(nvec, shift, r) >> shift))

    def global_index(self, slot, shift, r):
        q, w = slot >> shift, slot & ((1 << shift) - 1)
        return ((q * self.n + r) << shift) + w

    def oneshot_plan(self, count, es):
        n, epv = self.n, 16 // es
        nvec = cdiv(count, epv)
        shfl = n in (2, 4, 8) and nvec <= 4096
        blocks = self.grid_for(nvec * n, 1) if shfl else self.grid_for(nvec, 1)
        per_round = blocks * THREADS
        rounds = cdiv(count, per_round) + (cdiv(nvec * n, per_round) if shfl else 0) + 2
        return shfl, blocks, rounds


def unit_of(m):
    """with_unit: the widest access (16, 8, 4 or 1 bytes) dividing m."""
    return next(u for u in (16, 8, 4, 1) if m % u == 0)


def loop_passes(units, grid, per_cta):
    """Passes of each CTA of a grid-stride loop over `units` in which CTA b starts at b * per_cta and
    steps by grid * per_cta: the iterations in which its first thread still has work."""
    return [max(0, cdiv(units - b * per_cta, grid * per_cta)) for b in range(grid)]


# The kernels, each as loop(rules, count, es) -> (units of the busiest rank, grid, per_cta, lane):
# the busiest rank's loop runs over `units`, CTA b from b * per_cta, one UNROLL slot is `lane` units
# wide.  Counts are elements of es bytes; the reduction kernels take 16-byte-aligned buffers (their
# vector loop), the byte-moving ones their widest access unit.
def _owner(R, count, es, min_shift=0):
    epv = 16 // es
    nh = cdiv(count, epv)  # the host's vector count; the kernels use whole vectors only
    sh = R.own_shift(nh, min_shift)
    return count // epv, sh, cdiv(nh, R.n)


def loop_twoshot(R, count, es):
    nvec, sh, per = _owner(R, count, es)
    _, u = R.tiling(es)
    return max(R.owned(nvec, sh, r) for r in range(R.n)), R.grid_for(per, u), THREADS * u, THREADS


loop_scan = loop_twoshot  # launch_scan: the same ownership, tiling and grid


def loop_ring(R, count, es):
    epv = 16 // es
    groups = count // epv
    return cdiv(groups, R.n), R.grid_for(cdiv(cdiv(count, epv), R.n), 4), THREADS, THREADS


def loop_oneshot(R, count, es):
    """Both forms: the shuffle form's CTA b starts at vector b * 512 / n and a round covers
    grid * 512 / n vectors; the rank-order form's CTA b at b * 512."""
    shfl, blocks, _ = R.oneshot_plan(count, es)
    per = THREADS // R.n if shfl else THREADS
    return count // (16 // es), blocks, per, per


def loop_ll(R, count, es):
    ncell = cdiv(count * es, 8)
    return ncell, int(max(1, min(cdiv(ncell, LL_THREADS), LL_CTAS))), LL_THREADS, LL_THREADS


def loop_reduce_scatter(R, count, es):
    epv = 16 // es
    return count // epv, R.grid_for(cdiv(count, epv), 2), THREADS * 2, THREADS


def loop_bcast(R, count, es):
    b = count * es
    u = unit_of(b)
    return b // u, R.grid_for(b // 16 + 1, 4), THREADS * 4, THREADS


def loop_bcast2(R, count, es):
    """The two-shot Bcast: non-root k copies slice k of ceil(vectors / (n-1)) 16-byte granules."""
    b = count * es
    u = unit_of(b)
    nvec = b // 16 + 1
    per_b = cdiv(cdiv(b, 16), R.n - 1) * 16
    return min(per_b, b) // u, R.grid_for(nvec // (R.n - 1) + 1, 4), THREADS * 4, THREADS


loop_allgather = loop_bcast  # grid_for(bytes / 16 + 1, 4), copy_units<U, 4> over the rank's block
loop_alltoall = loop_bcast   # the same grid; push_rotated<U, 4> over each block in turn


def loop_allgather_ring(R, count, es):
    b = count * es
    u = unit_of(b)
    return b // u, R.grid_for(b // 16 + 1, 4), THREADS, THREADS


def loop_v(R, counts, es):
    """Gatherv, Scatterv and Allgatherv (vtable_grid): the largest block is the busiest loop."""
    big = max(counts) * es
    bits = 0
    for r in range(R.n + 1):
        bits |= sum(counts[:r]) * es  # vtable_bits: the displacements pick the access unit
    u = unit_of(bits)
    return big // u, R.grid_for(big // 16 + 1, 4), THREADS * 4, THREADS


def loop_alltoallv(R, counts, es):
    """Alltoallv: block_cap() CTAs whatever the table; counts is the matrix, the largest block busiest."""
    big = max(max(row) for row in counts) * es
    return big // unit_of(big), R.block_cap(), THREADS * 4, THREADS


def loop_rsv(R, counts, es):
    """ReduceScatterv with rank 0's block the largest (displacement 0, so no split16 head)."""
    u = 8 if es == 4 else 4
    big = max(counts) * es
    return big // 16, R.grid_for(big // 16 + 1, u), THREADS * u, THREADS


def loop_copy(R, count, es):
    """launch_copy (the copies of Send / Receive): 64 KiB per CTA pass, 16-byte vectors when both
    ends agree mod 16."""
    nbytes = count * es
    cap = R.cap if R.cap > 0 else R.sm_count
    grid = int(max(1, min(cdiv(nbytes, COPY_THREADS * COPY_UNROLL * 16), cap)))
    return nbytes // 16, grid, COPY_THREADS * COPY_UNROLL, COPY_THREADS


LOOPS = {"oneshot": loop_oneshot, "oneshot_shfl": loop_oneshot, "twoshot": loop_twoshot, "reduce": loop_twoshot, "ring": loop_ring, "ll": loop_ll,
         "reduce_scatter": loop_reduce_scatter, "scan": loop_scan, "exscan": loop_scan, "bcast": loop_bcast,
         "bcast2": loop_bcast2, "allgather": loop_allgather, "allgather_ring": loop_allgather_ring, "alltoall": loop_alltoall,
         "v": loop_v, "alltoallv": loop_alltoallv, "rsv": loop_rsv, "copy": loop_copy}


def passes(R, kernel, count, es):
    """[passes of CTA b of the busiest rank]; the last CTA makes the fewest."""
    units, grid, per_cta, _ = LOOPS[kernel](R, count, es)
    return loop_passes(units, grid, per_cta)


def smem_tiles(R, count, es):
    """The TMA two-shot: per rank, [(tiles processed, tiles skipped) of CTA b], and the vectors of
    the rank's last processed tile.  Tile t of a rank covers its local slots [256 t, 256 t + 256);
    CTA b takes t = b, b + grid, ... below slots / 256 and skips those that start past nvec."""
    epv = 16 // es
    nh = cdiv(count, epv)
    nvec = count // epv
    sh = R.own_shift(nh, 8)
    grid = int(max(1, min(cdiv(cdiv(nh, R.n) * 16, 4096), R.block_cap())))
    out = []
    for r in range(R.n):
        ntiles = R.owner_slots(nvec, sh, r) // TILE_VECS
        start = [R.global_index(t * TILE_VECS, sh, r) for t in range(ntiles)]
        ctas = [(sum(1 for t in range(b, ntiles, grid) if start[t] < nvec), sum(1 for t in range(b, ntiles, grid) if start[t] >= nvec))
                for b in range(grid)]
        live = [g for g in start if g < nvec]
        out.append({"shift": sh, "ctas": ctas, "last_tile": min(TILE_VECS, nvec - live[-1]) if live else 0})
    return grid, out


# ---- choosing counts ----------------------------------------------------------------------------
def owner_nvec(R, x, es, min_shift=0):
    """A whole-vector count whose busiest rank (rank 0) owns exactly x vectors below it: with blocks
    of B = 2^floor(log2 x) vectors every rank owns block r and rank 0 also the partial block n."""
    b = 1 << (x.bit_length() - 1)
    return R.n * b + (x - b)


def targets(grid, per_cta, lane, p):
    """Busiest-rank loop lengths: exactly p passes of every CTA; one unit more (CTA 0 makes p + 1);
    a last pass of the last CTA in which its last UNROLL slot holds only 7 threads' units."""
    step = grid * per_cta
    return {"exact": p * step, "plus1": p * step + 1, "partial": (p - 1) * step + (grid - 1) * per_cta + per_cta - lane + 7}


def tail(es):
    """The count % EPV tail every reduction count carries."""
    return max(1, 16 // es - 1) if es < 16 else 0


def plan(R, kernel, es, p=3):
    """{plan name: count} for which the busiest rank of `kernel` makes p passes per CTA (see targets).
    The reductions carry a count % EPV tail; the byte kernels get one more plan, 'tail', whose
    narrower access unit multiplies the passes."""
    n, epv = R.n, 16 // es
    cap = R.block_cap()
    out = {}
    if kernel in ("twoshot", "reduce", "scan", "exscan"):
        _, u = R.tiling(es)
        for name, x in targets(cap, THREADS * u, THREADS, p).items():
            out[name] = owner_nvec(R, x, es) * epv + tail(es)
    elif kernel == "ring":
        for name, x in targets(cap, THREADS, THREADS, p).items():
            out[name] = x * n * epv + tail(es)
    elif kernel == "oneshot":  # the rank-order form: above 4096 vectors in worlds of 2, 4 and 8
        q = max(p, 4096 // (cap * THREADS) + 1) if n in (2, 4, 8) else p
        for name, x in targets(cap, THREADS, THREADS, q).items():
            out[name] = x * epv + tail(es)
    elif kernel == "oneshot_shfl":
        per = THREADS // n
        for name, x in targets(cap, per, per, p).items():
            out[name] = x * epv + tail(es)
    elif kernel == "reduce_scatter":
        for name, x in targets(cap, THREADS * 2, THREADS, p).items():
            out[name] = x * epv + tail(es)
    elif kernel in ("bcast", "allgather", "alltoall", "allgather_ring", "bcast2"):
        per_cta = THREADS if kernel == "allgather_ring" else THREADS * 4
        for name, x in targets(cap, per_cta, THREADS, p).items():
            out[name] = x * (n - 1 if kernel == "bcast2" else 1) * 16 // es
        out["tail"] = out["exact"] + 1
    elif kernel == "copy":
        for name, x in targets(min(cap, R.sm_count), COPY_THREADS * COPY_UNROLL, COPY_THREADS, p).items():
            out[name] = x * 16 // es
    elif kernel == "ll":  # past 32768 cells: one cell more, and a partial second pass of every CTA
        cells = ll_cells(n)
        want = {"plus1": LL_CTAS * LL_THREADS + 1, "partial": LL_CTAS * LL_THREADS + (LL_CTAS - 1) * LL_THREADS + 7, "full": cells}
        out = {k: c * 8 // es for k, c in want.items() if c <= cells}
    else:
        raise ValueError(kernel)
    return out


def smem_plan(R, es):
    """TMA two-shot counts: T tiles for every CTA of rank 0 (T = 4, 2 * kSmemStages + 1 and 12), the
    last one 100 vectors long; with rank 0's second block partial, the tiles after it are skipped."""
    epv = 16 // es
    out = {}
    for t in (4, 2 * SMEM_STAGES + 1, 12):
        x = (t * R.block_cap() - 1) * TILE_VECS + 100
        out["tiles%d" % t] = owner_nvec(R, x, es, 8) * epv + tail(es)
    return out


def v_table(R, es, p=3):
    """A Gatherv / Scatterv / Allgatherv table whose rank 0 block makes p passes per CTA, the other
    blocks 5 + r elements; and an Alltoallv matrix whose block 0 -> n-1 does the same."""
    x = targets(R.block_cap(), THREADS * 4, THREADS, p)["exact"]
    big = x * 16 // es
    counts = [big] + [5 + r for r in range(1, R.n)]
    skew = [[3 + i + 2 * j for j in range(R.n)] for i in range(R.n)]
    skew[0][R.n - 1] = big
    return counts, skew


def rsv_table(R, es, p=3):
    u = 8 if es == 4 else 4
    x = targets(R.block_cap(), THREADS * u, THREADS, p)["partial"]
    return [x * (16 // es) + tail(es)] + [3 + r for r in range(1, R.n)]


def hybrid_grid(R, count, es, permille, nvls_unroll=2, nvls_max_blocks=48, p2p_blocks=0):
    """launch_allreduce_hybrid_t: (NVLS CTAs, P2P CTAs, P2P vectors) of the fused kernel, or None when
    the call goes to the plain NVLS kernel -- always under cap 1 and 2, since each part needs a CTA
    and the NVLS part at least one of its own."""
    n, epv = R.n, 16 // es
    nvec = count // epv
    p2p = int(nvec * permille / 1000.0)
    p2p = p2p // (n << 8) * (n << 8)
    split = nvec - p2p
    if split == 0 or p2p == 0:
        return None
    u = 4 if nvls_unroll == 4 else 2
    nb_nvls = R.grid_for(cdiv(split, n), u)
    if R.cap <= 0:
        nb_nvls = min(nb_nvls, nvls_max_blocks)
    nb_p2p = p2p_blocks if p2p_blocks > 0 else R.block_cap() - nb_nvls
    nb_p2p = max(1, min(nb_p2p, R.block_cap() - nb_nvls))
    if nb_nvls + nb_p2p > R.block_cap():
        return None
    return nb_nvls, nb_p2p, p2p


HYBRID_PERMILLE = 800


def hybrid_plan(R, es, nvls_unroll=2):
    """A count at which, with HYBRID_PERMILLE of the message on the P2P side, the NVLS part fills two
    CTAs of 512 * u vectors per rank and the P2P part (the two-shot body) runs on the rest of the
    grid: five such shares per rank in all, four of them P2P."""
    u = 4 if nvls_unroll == 4 else 2
    return 5 * 1024 * u * R.n * (16 // es) + tail(es)


# ---- the GPU worker -------------------------------------------------------------------------------
def _gpu_imports():
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    global F, RW, SW, W, L, O, mpi, ALGOS
    import _footprint_worker as F  # noqa: E402
    import _rsv_worker as RW  # noqa: E402
    import _scan_worker as SW  # noqa: E402
    import _worker as W  # noqa: E402
    from _worker import ALGOS, L, O, mpi  # noqa: E402


ES = {"u8": 1, "f32": 4, "f64": 8, "i64": 8}
RED = ("f32", "f64", "i64")


class Tally:
    """What the planned calls reached.  Per kernel: the fewest passes per CTA on the busiest rank over
    its planned calls (TMA: tiles per CTA, per plan), and every (plan, dtype) that ran on 16-byte
    aligned heap buffers -- the only layout on which the vector and TMA loops run; the unaligned and
    host calls on top of those are counted apart."""

    def __init__(self, R, cap):
        self.R, self.rules, self.cap = R, Rules(R.n, cap), cap
        self.min, self.tiles, self.ran, self.planned, self.extra = {}, {}, {}, {}, {}

    def plan(self, kernel, names, dtypes):
        self.planned[kernel] = sorted("%s/%s" % (p, d) for p in names for d in dtypes)

    def note(self, kernel, name, dn, count):
        es = ES[dn]
        self.ran.setdefault(kernel, set()).add("%s/%s" % (name, dn))
        if kernel == "smem":
            _, per_rank = smem_tiles(self.rules, count, es)
            t = max(min(c[0] for c in r["ctas"]) for r in per_rank)
            self.tiles[name] = min(self.tiles.get(name, t), t)
        else:
            t = passes(self.rules, kernel, count, es)[-1]
        self.min[kernel] = min(self.min.get(kernel, t), t)

    def other(self, kernel, what):
        self.extra.setdefault(kernel, []).append(what)

    def report(self):
        return {"min_passes": self.min, "smem_tiles": self.tiles, "planned": self.planned,
                "ran_aligned": {k: sorted(v) for k, v in self.ran.items()}, "extra": self.extra}


UNALIGNED = ("symmetric", "mixed", "split")


def run_kernel(R, T, kernel, plans, dtypes, call, per_rank=False):
    """Every plan of `kernel` in every dtype on aligned heap buffers, the ops in a Latin square over
    plans and dtypes; then one call per unaligned layout (scalar paths, narrower units) and one on
    host views (staged through the heap).  plans(es) -> {name: count}; call(dn, count, layout, op
    index, k, kind) makes one checked call, k numbering the calls of this kernel.  per_rank: a call's
    largest buffer holds n counts (Allgather, Alltoall, ReduceScatter); the host call takes the
    smallest planned count, so that it stays below the chunked host pipeline."""
    names = list(plans(4))
    T.plan(kernel, names, dtypes)
    k = 0
    for pi, name in enumerate(names):
        for di, dn in enumerate(dtypes):
            count = plans(ES[dn])[name]
            call(dn, count, "aligned", (pi + di) % 3, k, "heap")
            T.note(kernel, name, dn, count)
            k += 1
    for j, layout in enumerate(UNALIGNED):
        dn, name = dtypes[j % len(dtypes)], names[(j + 1) % len(names)]
        call(dn, plans(ES[dn])[name], layout, j, k, "heap")
        T.other(kernel, "%s/%s/%s" % (name, dn, layout))
        k += 1

    def nbytes(dn, name):
        count = plans(ES[dn])[name]
        return (sum(count) if isinstance(count, list) else count * (R.n if per_rank else 1)) * ES[dn]
    dn, name = min(((d, p) for p in names for d in dtypes), key=lambda x: nbytes(*x))
    assert nbytes(dn, name) < R.pipe_min, (kernel, dn, name)
    call(dn, plans(ES[dn])[name], "aligned", 1, k, "host")
    T.other(kernel, "%s/%s/host" % (name, dn))


def allreduce_call(R, algo, kernel, inplace_all=False):
    def call(dn, count, layout, oi, k, kind):
        R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
        used = R.lib.b200mpi_get_algo(L.COLL_ALLREDUCE, count, O.NP2DT[np.dtype(F.DTYPES[dn])])
        assert used == ALGOS[algo], "allreduce %s count=%d ran as %s" % (algo, count, L.ALGO_NAMES.get(used, used))
        F.do_allreduce(R, algo, dn, count, layout, F.OPS[oi][0], inplace_all or k % 2 == 1, kind, coll="allreduce:" + kernel)
    return call


def part_reductions(R, T):
    n, P = R.n, T.rules
    planner = lambda kernel: (lambda es: plan(P, kernel, es))  # noqa: E731
    run_kernel(R, T, "oneshot", planner("oneshot"), RED, allreduce_call(R, "oneshot", "oneshot", True))
    if n in (2, 4, 8):
        run_kernel(R, T, "oneshot_shfl", planner("oneshot_shfl"), RED, allreduce_call(R, "oneshot", "oneshot_shfl", True))
        run_kernel(R, T, "smem", lambda es: smem_plan(P, es), RED, allreduce_call(R, "smem", "smem"))
    run_kernel(R, T, "twoshot", planner("twoshot"), RED, allreduce_call(R, "twoshot", "twoshot"))
    run_kernel(R, T, "ring", planner("ring"), RED, allreduce_call(R, "ring", "ring"))
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)

    def reduce(dn, count, layout, oi, k, kind):
        F.do_reduce(R, dn, count, layout, F.OPS[oi][0], 1 + k % (n - 1), k % 2 == 1, kind)
    run_kernel(R, T, "reduce", planner("reduce"), RED, reduce)
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)

    def reduce_scatter(dn, count, layout, oi, k, kind):
        F.do_reduce_scatter(R, dn, count, layout, F.OPS[oi][0], k % 2 == 1, kind)
    run_kernel(R, T, "reduce_scatter", planner("reduce_scatter"), RED, reduce_scatter, per_rank=True)
    R.lib.b200mpi_set_algo(L.COLL_REDUCE_SCATTER, 0)
    for exclusive in (False, True):
        def scan(dn, count, layout, oi, k, kind, exclusive=exclusive):
            SW.do_footprint(R, dn, count, layout, F.OPS[oi][0], k % 2 == 1, kind, exclusive)
        run_kernel(R, T, "exscan" if exclusive else "scan", planner("scan"), RED, scan)

    def rsv(dn, counts, layout, oi, k, kind):
        RW.do_footprint(R, dn, counts, layout, F.OPS[oi][0], k % 2 == 1, kind)
    run_kernel(R, T, "rsv", lambda es: {"partial": rsv_table(P, es)}, RED, rsv)


def part_ll(R, T):
    """LL (its grid ignores the cap): past 32768 cells where the world's lanes allow it."""
    P = T.rules
    run_kernel(R, T, "ll", lambda es: plan(P, "ll", es), ("f32", "f64"), allreduce_call(R, "ll", "ll"))
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)


def part_bytes(R, T):
    n, P = R.n, T.rules
    planner = lambda kernel: (lambda es: plan(P, kernel, es))  # noqa: E731
    bytes_types = ("u8", "f32", "i64")
    for algo, kernel in (("oneshot", "bcast"), ("twoshot", "bcast2")):
        def bcast(dn, count, layout, oi, k, kind, algo=algo):
            F.do_bcast(R, algo, dn, count, layout, (k + n // 2) % n, kind)
        run_kernel(R, T, kernel, planner(kernel), bytes_types, bcast)
    R.lib.b200mpi_set_algo(L.COLL_BCAST, 0)
    for algo, kernel in (("oneshot", "allgather"), ("ring", "allgather_ring")):
        def allgather(dn, count, layout, oi, k, kind, algo=algo):
            F.do_allgather(R, algo, dn, count, layout, layout == "aligned" and k % 2 == 1, kind)
        run_kernel(R, T, kernel, planner(kernel), bytes_types, allgather, per_rank=True)
    R.lib.b200mpi_set_algo(L.COLL_ALLGATHER, 0)

    def alltoall(dn, count, layout, oi, k, kind):
        F.do_alltoall(R, dn, count, layout, kind)
    run_kernel(R, T, "alltoall", planner("alltoall"), bytes_types, alltoall, per_rank=True)


def part_v(R, T):
    """F.part_v on the planned tables (sized for u8: wider types make more passes); it runs every
    dtype on every layout, heap and host."""
    counts, skew = v_table(T.rules, 1)
    F.part_v(R, counts, skew)
    for dn in ("u8", "f32", "i64"):
        T.note("v", "exact", dn, counts)
        T.note("alltoallv", "exact", dn, skew)
    T.plan("v", ["exact"], ("u8", "f32", "i64"))
    T.plan("alltoallv", ["exact"], ("u8", "f32", "i64"))


def part_p2p(R, T):
    """Send / Receive between ranks 2k and 2k+1 at the copy's planned sizes, heap (both ends at the
    same residue mod 16, so the vector loop runs) and host, into a buffer 3 elements longer whose extra
    room must stay unwritten."""
    rank, n, P = R.rank, R.n, T.rules
    names = list(plan(P, "copy", 1))
    T.plan("copy", names, ("u8", "f32"))
    if rank >= n - n % 2:  # no partner: keep the call numbers (the seeds of inputs and offsets) in step
        R.call += 2 * 2 * len(names)
        return
    peer = rank ^ 1
    for dn in ("u8", "f32"):
        es = ES[dn]
        dt = F.DTYPES[dn]
        for ki, kind in enumerate(("heap", "host")):
            for pi, (name, count) in enumerate(plan(P, "copy", es).items()):
                call = R.next_call("p2p")
                off = 4 * ((pi + ki) % 3)
                x = F.gen_values(dt, 1, count, call * 2 + (rank & ~1))[0]
                what = "send/receive %s count=%d kind=%s offset=%d cap=%d ranks %d->%d" % (dn, count, kind, off, T.cap, rank & ~1, (rank & ~1) + 1)
                if rank % 2 == 0:
                    send = F.Guarded(kind, dt, count, off, rank, call, body=x)
                    mpi.Send(send.view, peer, 40)
                    F.check(send, what + " [send must be unchanged]")
                    send.free()
                else:
                    recv = F.Guarded(kind, dt, count + 3, off, rank, call)
                    got = mpi.Receive(recv.view, peer, 40)
                    assert len(got) == count, "%s: received %d elements" % (what, len(got))
                    recv.set_body(x)
                    F.check(recv, what + " [recv: message, then 3 elements that must not be written]")
                    recv.free()
                if kind == "heap":
                    T.note("copy", name, dn, count)
                else:
                    T.other("copy", "%s/%s/host" % (name, dn))


def part_nvls(R, T):
    """The switch paths of the footprint test under this cap, then the hybrid Allreduce at the count
    hybrid_plan picks.  Under caps 1 and 2 a hybrid request runs the NVLS kernel (the fused kernel
    needs a CTA for each part); under cap 3 the fused kernel runs, its P2P part on one CTA."""
    F.part_nvls(R)
    if not R.nvls or R.n not in (2, 4, 8):  # the hybrid form exists in worlds of 2, 4 and 8
        return
    P, lib = T.rules, R.lib
    saved = {k: L.get_param(k) for k in ("hybrid_p2p_permille", "hybrid_min_bytes", "nvls_min_ranks")}
    lib.b200mpi_set_param(b"hybrid_p2p_permille", HYBRID_PERMILLE)
    lib.b200mpi_set_param(b"hybrid_min_bytes", 0)
    lib.b200mpi_set_param(b"nvls_min_ranks", 2)
    u = L.get_param("nvls_unroll")
    for i, (dn, opname) in enumerate((("f32", "sum"), ("f64", "sum"), ("i64", "max"))):
        count = hybrid_plan(P, ES[dn], u)
        F.do_allreduce(R, "hybrid", dn, count, "aligned", opname, i == 1, "heap", coll="allreduce:hybrid")
        got = hybrid_grid(P, count, ES[dn], HYBRID_PERMILLE, u, L.get_param("nvls_max_blocks"), L.get_param("hybrid_p2p_blocks"))
        T.other("hybrid", "%s count=%d: %s" % (dn, count, "fused kernel, CTAs (nvls, p2p) = %s" % (got[:2],) if got else "NVLS kernel"))
    for k, v in saved.items():
        lib.b200mpi_set_param(k.encode(), v)
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)


PARTS = {"reductions": part_reductions, "ll": part_ll, "bytes": part_bytes, "v": part_v, "p2p": part_p2p, "nvls": part_nvls}
SETS = {"full": "reductions,ll,bytes,v,p2p", "reduced": "reductions,bytes,p2p", "nvls": "nvls"}


def scenario_passes(a):
    R = F.Run(argparse.Namespace(trim="edges"))
    out = {"caps": {}, "skipped": []}
    parts = SETS[a.set].split(",")
    for cap in (1, 3):
        assert R.lib.b200mpi_set_max_blocks(cap) == 0, L.last_error()
        T = Tally(R, cap)
        secs = {}
        for name in parts:
            if name == "ll" and cap != 1:
                continue  # the LL grid ignores the cap
            t0 = time.time()
            PARTS[name](R, T)
            mpi.Barrier()
            secs[name] = round(time.time() - t0, 2)
        out["caps"][str(cap)] = dict(T.report(), seconds=secs)
    R.lib.b200mpi_set_max_blocks(0)
    out.update(checked=R.call, by_part=R.done, nvls=R.nvls, skipped=sorted(R.skipped))
    return out


# ---- ranks whose grids differ -------------------------------------------------------------------
def grid_cases(n):
    """(name, coll, algo, kernel, dtype): the signed kernel families run with rank 0's grid smaller."""
    cases = [("allreduce twoshot", "allreduce", "twoshot", "twoshot", "f32"), ("allreduce ring", "allreduce", "ring", "ring", "f64"),
             ("bcast", "bcast", "twoshot", "bcast2", "u8"), ("reduce_scatter", "reduce_scatter", "twoshot", "reduce_scatter", "i64"),
             ("alltoallv", "alltoallv", None, "alltoallv", "f32")]
    if n in (2, 4, 8):
        cases.insert(2, ("allreduce smem", "allreduce", "smem", "smem", "f32"))
    return cases


def differ_call(R, coll, algo, dn, count, kind):
    """One call through the C ABI on guarded buffers; returns (rc, [buffers to check], cleanup)."""
    lib, rank, n = R.lib, R.rank, R.n
    dt = F.DTYPES[dn]
    mk = L.DEVICE if kind == "heap" else L.HOST
    dtc = O.NP2DT[np.dtype(dt)]
    call = R.next_call("grids:" + coll)
    if coll == "alltoallv":
        skew = count
        row, col = [skew[rank][j] for j in range(n)], [skew[i][rank] for i in range(n)]
        send = F.Guarded(kind, dt, sum(row), 16, rank, call, body=F.gen_values(dt, 1, sum(row), call * 8 + rank)[0])
        recv = F.Guarded(kind, dt, sum(col), 32, rank, call + 1)
        rc = lib.b200mpi_alltoallv(send.ptr(), (ctypes.c_size_t * n)(*row), recv.ptr(), (ctypes.c_size_t * n)(*col), dtc, mk)
        return rc, [send, recv]
    if coll == "bcast":
        buf = F.Guarded(kind, dt, count, 0, rank, call, body=F.gen_values(dt, n, count, call)[rank])  # a body of its own on every rank
        lib.b200mpi_set_algo(L.COLL_BCAST, ALGOS[algo])
        return lib.b200mpi_bcast(buf.ptr(), count, dtc, n - 1, mk), [buf]
    ns = count * n if coll == "reduce_scatter" else count
    send = F.Guarded(kind, dt, ns, 0, rank, call, body=F.gen_values(dt, n, ns, call)[rank])
    recv = F.Guarded(kind, dt, count, 16, rank, call + 1)
    if coll == "reduce_scatter":
        lib.b200mpi_set_algo(L.COLL_REDUCE_SCATTER, L.ALGO_TWOSHOT)
        return lib.b200mpi_reduce_scatter(send.ptr(), recv.ptr(), count, dtc, mpi.MAX, mk), [send, recv]
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
    return lib.b200mpi_allreduce(send.ptr(), recv.ptr(), count, dtc, mpi.SUM, mk), [send, recv]


def scenario_grids(a):
    """Rank 0 caps its grid at 1 CTA, the others at 3 (and rank n-1 of a world of 4 or more not at
    all): each signed call must end as B200MPI_ERR_PEER on every rank, write nothing (heap, and a
    staged host recv that must not be copied back), and advance the epoch by the same amount on
    every rank; then the same call with equal caps is checked in full.  The LL Allreduce, whose grid
    ignores the cap and which carries no signature, must succeed and match under different caps."""
    R = F.Run(argparse.Namespace(trim="edges"))
    lib, rank, n = R.lib, R.rank, R.n
    mine = 1 if rank == 0 else (0 if rank == n - 1 and n >= 4 else 3)
    wide = Rules(n, 3)
    steps, refused = [], []
    old_ll = L.get_param("ll_max_bytes")
    assert lib.b200mpi_set_param(b"ll_max_bytes", 0) == 0  # keep AUTO choices off the unsigned LL path
    for ci, (name, coll, algo, kernel, dn) in enumerate(grid_cases(n)):
        es = ES[dn]
        if kernel == "smem":
            count = smem_plan(wide, es)["tiles4"]
        elif kernel == "alltoallv":
            count = v_table(wide, es)[1]
        else:
            count = plan(wide, kernel, es)["exact"]
        for kind in ("heap", "host"):
            assert lib.b200mpi_set_max_blocks(mine) == 0
            e0 = L.get_param("epoch")
            rc, bufs = differ_call(R, coll, algo, dn, count, kind)
            e1 = L.get_param("epoch")
            what = "%s %s count=%s kind=%s cap=%d rank=%d" % (name, dn, "table" if kernel == "alltoallv" else count, kind, mine, rank)
            assert rc == L.ERR_PEER, "%s: rc %d, want B200MPI_ERR_PEER (%s)" % (what, rc, L.last_error())
            for b in bufs:
                F.check(b, what + " [must not be written by a refused call]")
                b.free()
            steps.append((e1 - e0) % (1 << 32))
            refused.append(what)
        assert lib.b200mpi_set_max_blocks(3) == 0
        # the same family with equal grids, checked in full
        if coll == "allreduce":
            F.do_allreduce(R, algo, dn, count, "aligned", "sum", False, "heap", coll="grids:after")
        elif coll == "bcast":
            F.do_bcast(R, algo, dn, count, "aligned", n - 1, "heap")
        elif coll == "reduce_scatter":
            F.do_reduce_scatter(R, dn, count, "aligned", "max", False, "heap")
        else:
            F.part_v(R, *v_table(wide, es))
    for c in (L.COLL_ALLREDUCE, L.COLL_BCAST, L.COLL_REDUCE_SCATTER):
        lib.b200mpi_set_algo(c, 0)
    assert lib.b200mpi_set_param(b"ll_max_bytes", old_ll) == 0
    # LL under different caps: no signature, a grid that ignores the cap
    assert lib.b200mpi_set_max_blocks(mine) == 0
    ll = 0
    for dn in ("f32", "f64"):
        for count in sorted(plan(Rules(n, 0), "ll", ES[dn]).values()):
            F.do_allreduce(R, "ll", dn, count, "aligned", "max", False, "heap", coll="grids:ll")
            ll += 1
    lib.b200mpi_set_max_blocks(0)
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
    mpi.Barrier()
    return {"checked": R.call, "by_part": R.done, "refused": refused, "epoch_steps": steps, "ll_under_different_caps": ll, "cap": mine}


if __name__ == "__main__":
    _gpu_imports()
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--set", default="full", choices=sorted(SETS))
    opts, rest = ap.parse_known_args(sys.argv[1:])
    sys.argv = [sys.argv[0]] + rest  # _worker.main parses the rest
    W.SCENARIOS["passes"] = lambda a: scenario_passes(opts)
    W.SCENARIOS["grids"] = lambda a: scenario_grids(opts)
    W.main()
