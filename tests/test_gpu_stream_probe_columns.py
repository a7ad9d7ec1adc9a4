"""The streaming join's positional path: exact partition counts, the probe columns scattered straight into their result
slots, and the probe that reads the key column back from the result.  Covered: every column count per side (1..4), 0 %,
~10 % and 100 % misses, several batches on one handle (both cursor slots), a partition holding 80 % of a batch (spread over
many probe CTAs by the work list), and segmented batches with device-resident counts.  Every case checks through
tq_join_stats[7] (probe launches: 6 per positional batch, 3 on the general partitioned path) that the positional path
ran, and compares the result with the CPU oracle."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import INT64, Chunk, Column, DeviceColumn, device_to_host
from tinysql_b200.executor import INNER_JOIN
from util import assert_same_multiset

pytestmark = pytest.mark.gpu

POS_LAUNCHES = 6        # k_pos_count, k_pos_bases, k_scatter_cols, k_probe_pos, k_hole_pads, k_hole_move_pads
N_BUILD = 300_000       # >= 2^18 rows: the streaming build and the partitioned probe


@pytest.fixture(autouse=True)
def _partitions(monkeypatch):
    # 4,000 build rows per partition: 128 partitions of the 300,000-row build side (the positional path needs pbits > 0)
    monkeypatch.setenv("TQ_JOIN_PART_ROWS", "4000")
    monkeypatch.delenv("TQ_JOIN_NO_FAST", raising=False)


def _build_cols(rng, nb):
    bk = rng.permutation(N_BUILD).astype(np.int64) * 3 + 11
    return [Column(INT64, bk)] + [Column(INT64, bk * (c + 5) - c) for c in range(1, nb)]


def _probe_keys(rng, bk, n, miss, hot=0.0):
    k = rng.choice(bk, n)
    m = rng.random(n) < miss
    k[m] = bk.max() + 1 + rng.integers(0, 1 << 30, int(m.sum()))       # keys the build side does not have
    if hot:
        k[rng.random(n) < hot] = bk[7]
    return k


def _probe_cols(k, first_id, np_):
    ids = np.arange(first_id, first_id + len(k), dtype=np.int64)
    return [Column(INT64, k)] + [Column(INT64, ids * (c + 2) + c) for c in range(1, np_)]


class _Join:
    """a join handle fed through the device-memory C-ABI: build, then probe batches; drained into host columns"""

    def __init__(self, lib, bcols, np_):
        self.lib, self.nb, self.np = lib, len(bcols), np_
        self.tb, self.tp = (C.c_int32 * self.nb)(*([1] * self.nb)), (C.c_int32 * np_)(*([1] * np_))
        self.k = (C.c_int32 * 1)(0)
        d = L.TQJoinDesc(0, 1, self.nb, self.tb, np_, self.tp, 1, self.k, self.k, 0, 0)
        self.h = C.c_void_p()
        L.check(lib.tq_join_create(C.byref(d), C.byref(self.h)))
        self.keep = []
        self.out = [[] for _ in range(self.nb + np_)]
        d_b = [DeviceColumn.from_host(c) for c in bcols]
        self.keep += d_b
        barr = (L.TQColumn * self.nb)(*[x.tq() for x in d_b])
        for i in range(self.nb):
            barr[i].null_bitmap = None
        L.check(lib.tq_join_put_build(self.h, barr, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(self.h))
        self.parts = self.stats()[2]

    def stats(self):
        st = (C.c_int64 * 8)()
        L.check(self.lib.tq_join_stats(self.h, st))
        return list(st)

    def put(self, pcols):
        d_p = [DeviceColumn.from_host(c) for c in pcols]
        self.keep += d_p
        parr = (L.TQColumn * self.np)(*[x.tq() for x in d_p])
        for i in range(self.np):
            parr[i].null_bitmap = None
        L.check(self.lib.tq_join_put_probe(self.h, parr, None, L.TQ_MEM_DEVICE))

    def put_segments(self, regions, cap):
        """regions: one list of np column arrays per region; each region is a device buffer of `cap` rows whose row
        count lives in device memory"""
        cols = (L.TQColumn * (self.np * len(regions)))()
        cnt_ptrs = (C.c_void_p * len(regions))()
        for g, arrs in enumerate(regions):
            m = len(arrs[0])
            for c, a in enumerate(arrs):
                region = np.zeros(cap, np.int64)
                region[:m] = a
                p = _dev(region)
                self.keep.append(p)
                cols[self.np * g + c].data, cols[self.np * g + c].length = p.value, m
            cp = _dev(np.array([m], np.uint64))
            self.keep.append(cp)
            cnt_ptrs[g] = cp.value
        L.check(self.lib.tq_join_put_probe_segments(self.h, len(regions), cols, cnt_ptrs, cap))

    def drain(self):
        out = (L.TQColumn * len(self.out))()
        n, eof = C.c_int64(0), C.c_int32(0)
        while True:
            L.check(self.lib.tq_join_next_device(self.h, out, C.byref(n), C.byref(eof)))
            if n.value == 0:
                return
            for c in range(len(self.out)):
                self.out[c].append(device_to_host(INT64, out[c].data, None, n.value).values)

    def finish(self):
        L.check(self.lib.tq_join_probe_eof(self.h))
        self.drain()
        st = self.stats()
        got = Chunk([Column(INT64, np.concatenate(c) if c else np.zeros(0, np.int64)) for c in self.out])
        return got, st

    def close(self):
        L.check(self.lib.tq_join_destroy(self.h))
        for x in self.keep:
            if isinstance(x, C.c_void_p):
                self.lib.tq_device_free(x)
            else:
                x.free()


def _dev(a):
    p = C.c_void_p()
    L.check(L.load().tq_device_alloc(max(a.nbytes, 8), C.byref(p)))
    if a.nbytes:
        L.check(L.load().tq_memcpy_h2d(p, a.ctypes.data, a.nbytes))
    return p


def _run(lib, bcols, np_, batches, segmented=()):
    """batches: probe column lists put one after another; segmented: (regions, cap) pairs put after them.  Returns the
    result, the stats and the probe columns of everything put, concatenated (the oracle's probe side)."""
    j = _Join(lib, bcols, np_)
    try:
        assert j.parts == 128, "the build did not take 128 partitions"
        launches0 = j.stats()[7]
        for pcols in batches:
            j.put(pcols)
        for regions, cap in segmented:
            j.put_segments(regions, cap)
        got, st = j.finish()
    finally:
        j.close()
    n_batches = len(batches) + len(segmented)
    assert st[7] - launches0 == POS_LAUNCHES * n_batches, "a probe batch left the positional path"
    probe = [np.concatenate([b[c].values for b in batches] + [r[c] for regions, _ in segmented for r in regions]) for c in range(np_)]
    return got, probe


def _want(bcols, probe):
    t = [INT64] * len(bcols), [INT64] * len(probe)
    return O.hash_join(INNER_JOIN, True, t[0], bcols, t[1], [Column(INT64, a) for a in probe], [0], [0])


@pytest.mark.parametrize("np_", [1, 2, 3, 4])
@pytest.mark.parametrize("nb", [1, 2, 3, 4])
def test_every_column_count(lib, nb, np_):
    """NP x NB probe / build columns, two batches (both cursor slots) with ~10 % misses"""
    rng = np.random.default_rng(100 * nb + np_)
    bcols = _build_cols(rng, nb)
    bk = bcols[0].values
    batches = [_probe_cols(_probe_keys(rng, bk, n, 0.1), first, np_) for n, first in ((400_000, 0), (350_001, 400_000))]
    got, probe = _run(lib, bcols, np_, batches)
    assert_same_multiset(got, _want(bcols, probe))


@pytest.mark.parametrize("miss", [0.0, 0.1, 1.0])
def test_miss_fractions(lib, miss):
    """0 % misses (only the partition pads are holes: k_hole_pads), ~10 % and 100 % (the validity bitmap's holes), three
    batches on one handle"""
    rng = np.random.default_rng(int(miss * 10) + 7)
    bcols = _build_cols(rng, 2)
    bk = bcols[0].values
    batches, first = [], 0
    for n in (600_000, 123_457, 500_000):
        batches.append(_probe_cols(_probe_keys(rng, bk, n, miss), first, 2))
        first += n
    got, probe = _run(lib, bcols, 2, batches)
    want = _want(bcols, probe)
    if miss == 0.0:
        assert got.num_rows() == len(probe[0])
    if miss == 1.0:
        assert want.num_rows() == 0
    assert_same_multiset(got, want)


def test_hot_partition_spread_over_many_ctas(lib):
    """80 % of a 3,000,000-row batch carry one key: its partition holds ~2.4 M rows, ~290 probe CTAs of 11 tiles each"""
    rng = np.random.default_rng(5)
    bcols = _build_cols(rng, 2)
    bk = bcols[0].values
    batches = [_probe_cols(_probe_keys(rng, bk, 3_000_000, 0.05, hot=0.8), 0, 2), _probe_cols(_probe_keys(rng, bk, 200_000, 0.05), 3_000_000, 2)]
    got, probe = _run(lib, bcols, 2, batches)
    assert_same_multiset(got, _want(bcols, probe))


@pytest.mark.parametrize("np_", [2, 3])
def test_segmented_batches(lib, np_):
    """tq_join_put_probe_segments with device-resident counts: a skewed batch of 3 regions (80 % one key), then an ordinary
    batch and a second segmented batch on the same handle"""
    rng = np.random.default_rng(40 + np_)
    bcols = _build_cols(rng, 2)
    bk = bcols[0].values
    first = 0

    def region(n, hot):
        nonlocal first
        cols = [c.values for c in _probe_cols(_probe_keys(rng, bk, n, 0.09, hot=hot), first, np_)]
        first += n
        return cols
    seg1 = ([region(170_000, 0.8), region(200_000, 0.8), region(110_000, 0.8)], 200_000)
    plain = _probe_cols(_probe_keys(rng, bk, 300_000, 0.09), 10_000_000, np_)
    seg2 = ([region(90_000, 0.0), region(150_000, 0.0)], 160_000)
    got, probe = _run(lib, bcols, np_, [plain], segmented=[seg1, seg2])
    assert_same_multiset(got, _want(bcols, probe))
