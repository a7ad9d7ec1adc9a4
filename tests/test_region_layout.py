"""CPU suite: dist.RegionLayout, the one place that says where the region exchange's slots and regions sit and builds the
argument tables of the C calls from it.  RegionExchange, RegionJoin, RegionAgg and the emulated-rank tests all run on it;
here it is checked on its own, with host memory standing in for the receive buffers."""
import ctypes as C
import itertools

import numpy as np
import pytest

from tinysql_b200 import _lib as L
from tinysql_b200.dist import RegionLayout

TABLES = [[(3, 4096)], [(2, 12_288), (3, 4096), (3, 4096), (1, 8192)], [(4, 5), (1, 1), (2, 70_001)]]


class _HostLib:
    """the one library call RegionLayout makes itself, on host memory"""

    @staticmethod
    def tq_memcpy_d2h(dst, src, nbytes):
        C.memmove(dst, src.value if isinstance(src, C.c_void_p) else src, nbytes)
        return L.TQ_OK


def _parent_offsets(world, tables):
    """RegionExchange's layout before RegionLayout existed (caps already rounded): slot (t, src) at (t * world + src) * 16,
    the regions from the first page boundary after the slots, table after table, [src][col] x cap rows"""
    slot = {(t, s): (t * world + s) * 16 for t in range(len(tables)) for s in range(world)}
    off = ((len(tables) * world * 16 + 4095) // 4096) * 4096
    region = {}
    for t, (nc, cap) in enumerate(tables):
        for s in range(world):
            for c in range(nc):
                region[(t, s, c)] = off + ((s * nc + c) * cap) * 8
        off += world * nc * cap * 8
    return slot, region, off


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("pad_rows", [0, 64])
@pytest.mark.parametrize("ti", range(len(TABLES)))
def test_layout_disjoint_and_inside(world, pad_rows, ti):
    """no two regions overlap, nor a region and the slot block; every region (and its pad rows) ends inside bytes; the slot
    block and bytes are page-aligned; destinations differ only by their base"""
    tables = TABLES[ti]
    lay = RegionLayout(None, L, world, tables, pad_rows)
    base = 1 << 40
    lay.bases = [base + d * lay.bytes for d in range(world)]
    assert lay.bytes % 4096 == 0 and lay.reg_off[0] % 4096 == 0
    slot_end = len(tables) * world * 16
    assert lay.reg_off[0] >= slot_end
    slots = sorted(lay.slot_ptr(0, t, s) - base for t in range(len(tables)) for s in range(world))
    assert slots == list(range(0, slot_end, 16)), "the slots are not one dense block from offset 0"
    spans = []
    for t, (nc, cap) in enumerate(tables):
        for s, c in itertools.product(range(world), range(nc)):
            lo = lay.region_ptr(0, t, s, c) - base
            spans.append((lo, lo + (cap + pad_rows) * 8))
            for d in range(world):
                assert lay.region_ptr(d, t, s, c) - lay.bases[d] == lo
                assert lay.slot_ptr(d, t, s) - lay.bases[d] == lay.slot_ptr(0, t, s) - base
    spans.sort()
    assert spans[0][0] >= slot_end, "a region overlaps the slot block"
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), "two regions overlap"
    assert spans[-1][1] <= lay.bytes, "a region ends past the receive buffer"


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("ti", range(len(TABLES)))
def test_layout_without_padding_is_the_exchange_layout(world, ti):
    """pad_rows = 0 puts every slot and region where RegionExchange always put them, in a buffer of the same size"""
    tables = [(nc, (cap + 4095) // 4096 * 4096) for nc, cap in TABLES[ti]]
    lay = RegionLayout(None, L, world, tables)
    lay.bases = [0] * world
    slot, region, total = _parent_offsets(world, tables)
    assert {k: lay.slot_ptr(0, *k) for k in slot} == slot
    assert {k: lay.region_ptr(0, *k) for k in region} == region
    assert lay.bytes == total


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("pad_rows", [0, 64])
def test_layout_tables_in_c_order(world, pad_rows):
    """push_tables: dest_data[q * nw + c] = source src's region of column c on destination q, dest_counts[q] = its slot
    there; region_table: regions[g * nw + c] = destination dst's region of source g, column c, length = cap; count_ptrs[g]
    = source g's slot on dst"""
    tables = TABLES[1]
    lay = RegionLayout(None, L, world, tables, pad_rows)
    lay.bases = [(1 << 40) + d * lay.bytes for d in range(world)]
    for t, (nw, cap) in enumerate(tables):
        for x in range(world):
            dest, cnts = lay.push_tables(t, x)
            assert len(dest) == world * nw and len(cnts) == world
            regs, ptrs = lay.region_table(x, t), lay.count_ptrs(x, t)
            assert len(regs) == world * nw and len(ptrs) == world
            for q, c in itertools.product(range(world), range(nw)):
                assert dest[q * nw + c] == lay.region_ptr(q, t, x, c)
                assert regs[q * nw + c].data == lay.region_ptr(x, t, q, c)
                assert regs[q * nw + c].length == cap and not regs[q * nw + c].null_bitmap and not regs[q * nw + c].offsets
            for q in range(world):
                assert cnts[q] == lay.slot_ptr(q, t, x)
                assert ptrs[q] == lay.slot_ptr(x, t, q)


def test_layout_slot_reads_and_overflow():
    """read_slots returns {rows, epoch} per (table, source) of one destination; counts raises when a count passes its
    table's cap, which is what an overflowed push (~0) publishes"""
    world, tables = 3, [(2, 100), (1, 50), (3, 70)]
    lay = RegionLayout(_HostLib, L, world, tables)
    bufs = [np.zeros(lay.bytes // 8, np.uint64) for _ in range(world)]
    lay.bases = [b.ctypes.data for b in bufs]
    for d, t, s in itertools.product(range(world), range(len(tables)), range(world)):
        k = (lay.slot_ptr(d, t, s) - lay.bases[d]) // 8
        bufs[d][k:k + 2] = [10 * d + 3 * t + s, 40 + t]
    raw = lay.read_slots(1)
    assert raw.shape == (len(tables), world, 2)
    assert [[tuple(map(int, r)) for r in tab] for tab in raw] == [[(10 + 3 * t + s, 40 + t) for s in range(world)] for t in range(len(tables))]
    assert lay.counts(2, 1, 1) == [[23, 24, 25]]
    assert lay.counts(0) == [[3 * t + s for s in range(world)] for t in range(len(tables))]
    k = (lay.slot_ptr(0, 2, 1) - lay.bases[0]) // 8
    bufs[0][k] = np.uint64((1 << 64) - 1)
    assert lay.counts(0, 0, 2) == [[0, 1, 2], [3, 4, 5]], "only the tables asked for are read"
    with pytest.raises(RuntimeError, match="region overflow in table 2"):
        lay.counts(0)
