"""The harness of tests/test_gpu_footprint.py, checked without a GPU: the guarded-buffer layout, the
checker that reads it, the value generator, and the oracle's MAX / MIN orders on hand-worked vectors
whose answers differ between rank, tree and ring order."""
import numpy as np
import pytest

import _footprint_worker as F
from oracle import oracle as O

COUNTS = (0, 1, 3, 5, 7, 257, 4097)
WORLDS = (2, 3, 4, 6, 8)


def bits(x):
    x = np.asarray(x)
    return x.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[x.dtype.itemsize])


@pytest.mark.parametrize("dn", list(F.DTYPES))
def test_guard_layout_never_lets_a_view_overlap_its_guards(dn):
    dt = np.dtype(F.DTYPES[dn])
    res = F.RESIDUES[dt]
    for layout in F.LAYOUTS:
        for n in WORLDS:
            for key in range(12):
                offs = F.layout_offsets(layout, dt, n, key)
                assert len(offs) == n
                rs = [(s % 16, r % 16) for s, r in offs]
                assert all(a in res and b in res for a, b in rs), (layout, rs)
                if layout == "aligned":
                    assert all(a == 0 and b == 0 for a, b in rs)
                elif layout == "symmetric":
                    assert len(set(offs)) == 1 and rs[0][0] != 0 and rs[0][0] == rs[0][1]
                elif layout == "mixed":
                    assert all(rs[r][0] != rs[(r + 1) % n][0] for r in range(min(n, len(res)) - 1)), rs
                else:
                    assert all(a != b for a, b in rs), rs
                for count in COUNTS:
                    for off in {o for pair in offs for o in pair}:
                        head, body, tail, total = F.zones(count, dt, off)
                        assert head >= F.GUARD and tail >= F.GUARD and head + body + tail == total
                        assert head % dt.itemsize == 0 and head % 16 == off % 16 and total % 16 == 0
                        g = F.Guarded("host", dt, count, off, 1, key)
                        assert g.mem.ctypes.data % 64 == 0 and g.mem.size == total
                        assert g.view.nbytes == body == count * dt.itemsize
                        if count:  # an empty view is passed as NULL
                            assert g.view.ctypes.data - g.mem.ctypes.data == head
                        assert not np.isin(g.image[:head], F.NOT_WRITTEN).any()
                        assert not np.isin(g.image[head + body:], F.NOT_WRITTEN).any()


def test_guard_pattern_depends_on_rank_and_call():
    a = F.guard_pattern(0, 5, 256)
    assert not np.array_equal(a, F.guard_pattern(1, 5, 256))
    assert not np.array_equal(a, F.guard_pattern(0, 6, 256))
    assert not np.isin(np.concatenate([F.guard_pattern(r, c, 4096) for r in range(8) for c in range(64)]), F.NOT_WRITTEN).any()


@pytest.mark.parametrize("dn", ["u8", "f32", "f64", "i64"])
def test_checker_names_the_first_differing_byte_and_its_side(dn):
    dt = F.DTYPES[dn]
    g = F.Guarded("host", dt, 257, 8, 0, 3, body=F.gen_values(dt, 1, 257, 3)[0])
    F.check(g, "clean")
    for pos, side in ((g.head - 1, "head guard"), (g.head, "body byte 0 "), (g.head + g.nbody, "tail guard byte 0 "),
                      (g.total - 1, "tail guard")):
        saved = g.mem[pos]
        g.mem[pos] ^= 0x10
        for mode in ("exact", "sum"):
            with pytest.raises(AssertionError, match=side):
                F.check(g, "one byte flipped", mode)
        g.mem[pos] = saved
    F.check(g, "restored")


def test_sum_mode_compares_nan_positions_not_payloads():
    g = F.Guarded("host", np.float32, 4, 4, 0, 1, body=np.array([1.0, np.nan, -0.0, 2.0], dtype=np.float32))
    g.view[1] = F._qnan(np.float32, 0x3)  # another NaN payload: fine for a sum
    F.check(g, "sum", "sum")
    with pytest.raises(AssertionError):
        F.check(g, "max", "exact")
    g.view[2] = 0.0  # +0 for -0 is a wrong sum (the sign is the element's last byte)
    with pytest.raises(AssertionError, match=r"body byte 11 \(element 2\)"):
        F.check(g, "sum", "sum")


@pytest.mark.parametrize("dn", ["f32", "f64", "i64"])
def test_generator_places_every_special_first_in_the_middle_and_last(dn):
    dt = F.DTYPES[dn]
    for n in (3, 4, 6, 8):
        for count in (3 * len(F.specials(dt, 0)), 257, 4097):
            xs = F.gen_values(dt, n, count, count + n)
            for k in range(len(F.specials(dt, 0))):
                held = {r for r in range(n) if (bits(xs[r]) == bits(F.specials(dt, r)[k])).any()}
                assert 0 in held and n - 1 in held and held & set(range(1, n - 1)), (dn, n, count, k, held)


def test_generator_values_are_signed_and_span_a_wide_range():
    for dt, span in ((np.float32, 40), (np.float64, 120)):
        x = np.concatenate(F.gen_values(dt, 4, 4097, 9))
        fin = x[np.isfinite(x) & (x != 0)]
        assert 0.3 < np.mean(fin < 0) < 0.7
        e = np.frexp(fin)[1]
        assert e.max() - e.min() > span
        assert np.signbit(x[x == 0]).any() and (~np.signbit(x[x == 0])).any()
    x = np.concatenate(F.gen_values(np.int64, 4, 4097, 9))
    for v in (np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0):
        assert (x == v).any()
    assert (x < -(1 << 62)).any() and (x > (1 << 62)).any()


NAN = np.float32(np.nan)
NZ = np.float32(-0.0)

# (n, op, group, values of ranks 0..n-1 at one element, {order: answer}).  MAX is b > a ? b : a and
# MIN b < a ? b : a: a NaN or a zero of the other sign on the right loses, on the left it stays.
# count = 4n f32 elements, so the ring's chunk c is group c and starts at rank c.
HAND = [
    (4, O.MAX, 0, [1, 2, NAN, 3], {O.ORDER_RANK: 3, O.ORDER_TREE: 2, O.ORDER_RING: 3}),
    (4, O.MAX, 1, [1, NAN, 2, 3], {O.ORDER_RANK: 3, O.ORDER_TREE: 3, O.ORDER_RING: NAN}),
    (4, O.MAX, 1, [0.0, NZ, -1, -1], {O.ORDER_RANK: 0.0, O.ORDER_TREE: 0.0, O.ORDER_RING: NZ}),
    (4, O.MIN, 0, [1, 2, NAN, 0], {O.ORDER_RANK: 0, O.ORDER_TREE: 1, O.ORDER_RING: 0}),
    (4, O.MIN, 2, [1, 1, 0.0, NZ], {O.ORDER_RANK: 0.0, O.ORDER_TREE: 0.0, O.ORDER_RING: 0.0}),
    (4, O.MIN, 3, [1, 1, 0.0, NZ], {O.ORDER_RANK: 0.0, O.ORDER_TREE: 0.0, O.ORDER_RING: NZ}),
    (8, O.MAX, 0, [1, 2, 3, 4, NAN, 5, 6, 7], {O.ORDER_RANK: 7, O.ORDER_TREE: 4, O.ORDER_RING: 7}),
    (8, O.MAX, 4, [1, 2, 3, 4, NAN, 5, 6, 7], {O.ORDER_RANK: 7, O.ORDER_TREE: 4, O.ORDER_RING: NAN}),
    (8, O.MAX, 3, [0.0, -1, -1, NZ, -1, -1, -1, -1], {O.ORDER_RANK: 0.0, O.ORDER_TREE: 0.0, O.ORDER_RING: NZ}),
    (8, O.MIN, 6, [NZ, 1, 1, 1, 1, 1, 0.0, 1], {O.ORDER_RANK: NZ, O.ORDER_TREE: NZ, O.ORDER_RING: 0.0}),
    (8, O.MIN, 0, [1, 2, 3, 4, NAN, 0, 0, 0], {O.ORDER_RANK: 0, O.ORDER_TREE: 1, O.ORDER_RING: 0}),
    (8, O.MIN, 1, [1, NAN, 1, 1, 1, 1, 1, 0], {O.ORDER_RANK: 0, O.ORDER_TREE: 0, O.ORDER_RING: NAN}),
]


@pytest.mark.parametrize("case", range(len(HAND)))
def test_oracle_max_min_orders_on_hand_worked_vectors(case):
    n, op, group, vals, answers = HAND[case]
    count = 4 * n
    xs = [np.full(count, 0.5 + r, dtype=np.float32) for r in range(n)]
    e = 4 * group + 1
    for r in range(n):
        xs[r][e] = vals[r]
    for order, want in answers.items():
        got = O.allreduce(xs, op=op, order=order)
        assert bits(got[e]) == bits(np.float32(want)), (order, got[e], want)
        assert bits(O.allreduce_np(xs, op=op, order=order)[e]) == bits(np.float32(want)), order


def test_hand_worked_vectors_tell_every_pair_of_orders_apart():
    """Across the table, for each of MAX and MIN in worlds of 4 and 8, some vector's answer differs
    between rank and tree order and some between rank and ring order."""
    for n in (4, 8):
        for op in (O.MAX, O.MIN):
            rows = [a for m, o, _, _, a in HAND if m == n and o == op]
            for other in (O.ORDER_TREE, O.ORDER_RING):
                assert any(bits(np.float32(a[O.ORDER_RANK])) != bits(np.float32(a[other])) for a in rows), (n, op, other)


@pytest.mark.parametrize("n", [4, 8])
@pytest.mark.parametrize("dn", ["f32", "f64"])
def test_generated_inputs_tell_the_orders_apart(n, dn):
    """The GPU test's own inputs give different MAX and MIN bits in rank, tree and ring order, so a
    kernel that reduces in another order than its own fails there."""
    dt = F.DTYPES[dn]
    xs = F.gen_values(dt, n, 4097, 11)
    for op in (O.MAX, O.MIN):
        rank = bits(O.allreduce(xs, op=op, order=O.ORDER_RANK))
        for other in (O.ORDER_TREE, O.ORDER_RING):
            assert (rank != bits(O.allreduce(xs, op=op, order=other))).any(), (op, other)


@pytest.mark.parametrize("dn", ["f32", "f64"])
def test_tolerance_mode_on_an_in_place_reduce_scatter_buffer(dn):
    """In place, ReduceScatter's send holds n blocks and only the own block is reduced: under the switch's
    tolerance that block is compared within 1e-6 * sum_r |x_r|, every other element byte for byte."""
    dt = F.DTYPES[dn]
    n, count, rank = 4, 4099, 1
    ins = F.gen_values(dt, n, count * n, 21)
    blocks = [x[rank * count:(rank + 1) * count] for x in ins]
    want = O.reduce_scatter(ins, rank, order=O.ORDER_F64)
    g = F.Guarded("host", dt, count * n, 4 if dn == "f32" else 8, rank, 21, body=ins[rank])
    g.set_body(want, rank * count)
    g.load()
    F.check(g, "oracle answer", "tol", blocks, lo=rank * count)
    # a result one ulp off inside the own block is within the tolerance
    i = int(np.flatnonzero(np.isfinite(want) & (np.abs(want) > 1))[0])
    g.view[rank * count + i] = np.nextafter(want[i], np.inf, dtype=dt)
    F.check(g, "one ulp off", "tol", blocks, lo=rank * count)
    # far off inside the block fails, named as a body element of the own block
    g.view[rank * count + i] = want[i] * 2
    with pytest.raises(AssertionError, match="element %d\\)" % (rank * count + i)):
        F.check(g, "twice the sum", "tol", blocks, lo=rank * count)
    g.view[rank * count + i] = want[i]
    # outside the own block nothing may change, not even the sign of a zero
    j = int(np.flatnonzero(ins[rank][:count] == 0)[0])
    g.view[j] = -g.view[j]
    with pytest.raises(AssertionError, match="element %d\\)" % j):
        F.check(g, "send block 0 touched", "tol", blocks, lo=rank * count)
    g.view[j] = ins[rank][j]
    F.check(g, "restored", "tol", blocks, lo=rank * count)


def test_options_default_to_every_part_at_full_counts():
    opts, rest = F.parse_options(["--trim", "edges", "--out", "x"])
    assert opts.trim == "edges" and rest == ["--out", "x"]
    opts, _ = F.parse_options([])
    assert opts.parts.split(",") == list(F.PARTS) and opts.trim == "full"


def test_edge_counts_keep_both_one_shot_forms():
    """Worlds of 8 run the shuffle one-shot (<= 4096 vectors) and the rank-order one above it."""
    for dt in (np.float32, np.float64, np.int64):
        e = F.epv(dt)
        counts = F.counts_for(dt, F.allreduce_passes("oneshot", 8, dt), "edges")
        assert any(-(-c // e) <= 4096 for c in counts) and any(-(-c // e) > 4096 for c in counts), counts
