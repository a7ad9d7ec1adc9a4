"""The streaming join's paged positional result at its page edges.  The probe scatter hands out result pages of PAGE slots
while it runs, one partition per page, and the holes are the unfilled tails of the partitions' last pages.  Probe keys are
aimed at chosen partitions (hash_targets: the partition of a key is the top pbits bits of tqd::hash_key), and every case
asserts that its batch really has the partition sizes it is about: exact multiples of PAGE and one row either side, every
partition ending on a page boundary (no holes at all), fewer rows than partitions, one row, all rows in one partition (the
longest page-table row), several batches on one handle whose page-table rows differ (a stale entry of an earlier batch would
misplace rows), segmented batches, and every column count per side.  Each batch must run on the positional path (6 probe
launches: k_pos_reset, k_scatter_cols, k_pos_pages, k_probe_pos, k_hole_pages, k_hole_move_pages) and the result must equal
the CPU oracle's."""
import numpy as np
import pytest

import hash_targets as HT
from test_gpu_stream_probe_columns import _build_cols, _probe_cols, _run, _want
from util import assert_same_multiset

pytestmark = pytest.mark.gpu

PBITS = 7
P = 1 << PBITS
PP_TILE_ROWS = 768


def page_rows(n, np_):
    """join_stream.cuh pos_page_rows at 128 partitions: whole probe tiles (768 rows), at least one scatter tile (4096 rows for
    one or two probe columns, else 2048), else as many tiles as keep P * page_rows within 1 % of the batch"""
    scatter_tile = 4096 if np_ <= 2 else 2048
    min_tiles = -(-scatter_tile // PP_TILE_ROWS)
    return max(n // (100 * P * PP_TILE_ROWS), min_tiles) * PP_TILE_ROWS


@pytest.fixture(autouse=True)
def _partitions(monkeypatch):
    # 4,000 build rows per partition: 128 partitions of the 300,000-row build side (the positional path needs pbits > 0)
    monkeypatch.setenv("TQ_JOIN_PART_ROWS", "4000")
    monkeypatch.delenv("TQ_JOIN_NO_FAST", raising=False)


def part_of(keys):
    return HT.table_of(HT.hash_key(np.asarray(keys, np.int64)), PBITS).astype(np.int64)


class Aim:
    """probe keys of the build side, by partition; keys past the build side's largest are misses"""

    def __init__(self, rng, bk):
        self.rng, self.bk = rng, bk
        pk = part_of(bk)
        self.by_part = [bk[pk == q] for q in range(P)]
        assert min(len(k) for k in self.by_part) > 0

    def keys(self, sizes, miss=0.0):
        """sizes: {partition: rows}; returns the keys shuffled, with `miss` of them replaced by absent keys"""
        k = np.concatenate([self.rng.choice(self.by_part[q], n) for q, n in sizes.items() if n] or [np.zeros(0, np.int64)])
        k = self.rng.permutation(k)
        m = self.rng.random(len(k)) < miss
        k[m] = self.bk.max() + 1 + self.rng.integers(0, 1 << 30, int(m.sum()))
        return k


def sizes_of(keys, bk):
    found = np.isin(keys, bk)
    return np.bincount(part_of(keys[found]), minlength=P)


def _setup(seed, nb=2):
    rng = np.random.default_rng(seed)
    bcols = _build_cols(rng, nb)
    return bcols, Aim(rng, bcols[0].values)


def _check(lib, bcols, np_, batches, segmented=()):
    got, probe = _run(lib, bcols, np_, batches, segmented)
    assert_same_multiset(got, _want(bcols, probe))
    return got


def _spread(rng, n, exclude=()):
    """n rows over the partitions not in `exclude`, at random"""
    parts = [q for q in range(P) if q not in exclude]
    c = np.bincount(rng.choice(len(parts), n), minlength=len(parts))
    return {q: int(x) for q, x in zip(parts, c)}


@pytest.mark.parametrize("delta", [-1, 0, 1])
@pytest.mark.parametrize("k", [1, 3])
def test_partition_at_page_multiples(lib, delta, k):
    """three partitions of exactly k * PAGE + delta rows in a batch of ~460,000"""
    bcols, aim = _setup(11 + 3 * k + delta)
    n = 460_000
    page = page_rows(n, 2)
    want = k * page + delta
    sizes = _spread(aim.rng, n - 3 * want, exclude=(5, 40, 127))
    sizes.update({5: want, 40: want, 127: want})
    keys = aim.keys(sizes)
    assert len(keys) == n and page_rows(len(keys), 2) == page
    got_sizes = sizes_of(keys, aim.bk)
    assert got_sizes[5] == got_sizes[40] == got_sizes[127] == want
    _check(lib, bcols, 2, [_probe_cols(keys, 0, 2)])


@pytest.mark.parametrize("pages_each", [1, 2])
def test_every_partition_ends_on_a_page_boundary(lib, pages_each):
    """every partition holds a whole number of pages: the result has no hole at all"""
    bcols, aim = _setup(21 + pages_each)
    page = page_rows(P * 4608 * pages_each, 2)
    assert page == 4608
    keys = aim.keys({q: page * pages_each for q in range(P)})
    assert page_rows(len(keys), 2) == page
    assert (sizes_of(keys, aim.bk) % page == 0).all()
    got = _check(lib, bcols, 2, [_probe_cols(keys, 0, 2)])
    assert got.num_rows() == len(keys)


@pytest.mark.parametrize("n", [1, 2, 100, 127])
def test_fewer_rows_than_partitions(lib, n):
    """1 .. 127 rows, in distinct partitions: as many pages as rows, each almost all hole"""
    bcols, aim = _setup(30 + n)
    keys = aim.keys({q: 1 for q in aim.rng.choice(P, n, replace=False)})
    assert len(keys) == n < P and sizes_of(keys, aim.bk).max() == 1
    _check(lib, bcols, 2, [_probe_cols(keys, 0, 2)])


@pytest.mark.parametrize("miss", [0.0, 0.1, 1.0])
def test_all_rows_in_one_partition(lib, miss):
    """1,000,000 rows of one partition: the longest page-table row (n / PAGE + 1 entries), one probe CTA after another on it"""
    bcols, aim = _setup(41 + int(miss * 10))
    keys = aim.keys({77: 1_000_000}, miss=miss)
    assert (part_of(keys[np.isin(keys, aim.bk)]) == 77).all()
    _check(lib, bcols, 2, [_probe_cols(keys, 0, 2)])


@pytest.mark.parametrize("miss", [0.0, 0.1, 1.0])
def test_miss_fractions_at_page_edges(lib, miss):
    """page-multiple partitions with 0 %, ~10 % and 100 % misses: the device hole runs (no miss) and the bitmap's holes"""
    bcols, aim = _setup(51 + int(miss * 10))
    n = 300_000
    page = page_rows(n, 2)
    sizes = _spread(aim.rng, n - 2 * page - 1, exclude=(0, 1))
    sizes.update({0: page, 1: page - 1})
    keys = aim.keys(sizes, miss=miss)
    if miss == 0.0:
        assert sizes_of(keys, aim.bk)[0] == page
    _check(lib, bcols, 2, [_probe_cols(keys, 0, 2)])


@pytest.mark.parametrize("np_", [1, 2, 3, 4])
@pytest.mark.parametrize("nb", [1, 2, 3, 4])
def test_every_column_count(lib, nb, np_):
    """NP x NB columns (three or four probe columns take 2048-row scatter tiles, hence smaller pages) with a partition of
    exactly one page and one of one page + 1 row"""
    bcols, aim = _setup(60 + 10 * nb + np_, nb)
    n = 200_000
    page = page_rows(n, np_)
    sizes = _spread(aim.rng, n - 2 * page - 1, exclude=(3, 4))
    sizes.update({3: page, 4: page + 1})
    keys = aim.keys(sizes, miss=0.02)
    _check(lib, bcols, np_, [_probe_cols(keys, 0, np_)])


def test_batches_on_one_handle_with_different_pages(lib):
    """five batches alternate the two cursor slots, and each slot's page table is reused with different rows: partition 9
    holds 60 pages, then 1 row, then 3 pages; partition 100 the opposite.  An entry of an earlier batch read as current
    would put rows on another batch's page."""
    bcols, aim = _setup(71)
    plans = [{9: 60 * 4608, 100: 1}, {9: 5, 100: 7}, {9: 1, 100: 60 * 4608 + 17}, {9: 2 * 4608, 100: 3}, {9: 3 * 4608, 100: 4608 - 1}]
    batches, first = [], 0
    for plan in plans:
        sizes = _spread(aim.rng, 20_000, exclude=(9, 100))
        sizes.update(plan)
        keys = aim.keys(sizes)
        assert page_rows(len(keys), 2) == 4608
        batches.append(_probe_cols(keys, first, 2))
        first += len(keys)
    _check(lib, bcols, 2, batches)


@pytest.mark.parametrize("np_", [2, 3])
def test_segmented_batches(lib, np_):
    """tq_join_put_probe_segments: regions whose partitions sit on page edges, then a plain batch, then one all-in-one-partition
    segmented batch"""
    bcols, aim = _setup(80 + np_)
    cap = 200_000
    n_all = 3 * ((cap + 4095) // 4096 * 4096)
    page = page_rows(n_all, np_)
    first = 0

    def region(sizes, miss=0.0):
        nonlocal first
        cols = [c.values for c in _probe_cols(aim.keys(sizes, miss), first, np_)]
        first += len(cols[0])
        return cols
    seg1 = ([region({2: page, 3: page + 1, 4: 50_000}), region({2: page, 5: 10_000}, miss=0.05), region({3: 1})], cap)
    plain = _probe_cols(aim.keys(_spread(aim.rng, 100_000)), 10_000_000, np_)
    seg2 = ([region({6: 150_000}), region({6: 120_000})], 160_000)
    _check(lib, bcols, np_, [plain], segmented=[seg1, seg2])
