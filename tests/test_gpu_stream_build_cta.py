"""The streaming build with each sub-table built in one CTA's shared memory (k_build_cta), against the CPU oracle: every
entry width, one and several sub-tables per scatter slab, the positional and the general probes, the shape that still
takes the cluster build, the hand-overs to the general build, and skewed slabs that stay on the CTA build.  Every case
asserts which build ran (tq_join_build_path).

hash_targets.stream_geometry restates the cluster build's sizing, which try_stream_build now uses only where no sub-table
size one CTA holds stays within 2^PART_MAX_BITS sub-tables; cta_geometry below restates the CTA build's.  The cluster build
(k_build_cluster, unchanged but for the row counter that now sets the table's row count) is covered here by the 1.2e7-row
cases; the aimed edge tests of test_gpu_hash_edges.py were written for its sizing and now mostly reach the CTA build."""
import ctypes as C

import numpy as np
import pytest

import hash_targets as H
import oracle_py as O
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import FLOAT64, INT64, Column
from tinysql_b200.executor import INNER_JOIN, LEFT_OUTER_JOIN, RIGHT_OUTER_JOIN, HashJoinExec, MockDataSource
from util import assert_same_multiset

pytestmark = pytest.mark.gpu

EMPTY_MARKER = np.int64(np.uint64(H.EMPTY_KEY).astype(np.int64))
BT_MAX_BYTES = 200 << 10  # one CTA's sub-table


def cta_geometry(n, nb, part_rows=H.PART_TARGET_ROWS):
    """try_stream_build's sizing when a sub-table fits one CTA (None when it does not: the cluster build takes it)"""
    pbits = 0
    while (part_rows << pbits) < n:
        pbits += 1
    pbits = min(pbits, H.SA_MAX_PBITS)
    shift = 2 if nb > 2 else 1
    for sbits in range(0, H.PART_MAX_BITS - pbits + 1):
        mean = n / float((1 << pbits) << sbits)
        est_max = int(mean + 8.0 * np.sqrt(mean) + 64.0)
        cap = (est_max * 100 // H.MAX_LOAD_PCT + 15) & ~15
        if (cap << shift) * 8 <= BT_MAX_BYTES:
            tbits = pbits + sbits
            bbits = min(tbits, H.SA_MAX_PBITS)
            return dict(pbits=pbits, tbits=tbits, bbits=bbits, lbits=tbits - bbits, cap=cap, max_rows=cap * H.MAX_LOAD_PCT // 100,
                        bin_slab=H.slab_rows(n, 1 << bbits, True))
    return None


# (build rows, TQ_JOIN_PART_ROWS) -> one sub-table per slab (1e6 rows: 2^8 of them, 2^9 for 32-byte entries), or several
# (4e6 rows: 2^10 sub-tables, 2 per slab; 2^11 for 32-byte entries, 4 per slab)
SHAPES = {"one_per_slab": (1_000_000, 150000), "several_per_slab": (4_000_000, 20000)}


def _switches(monkeypatch, part_rows):
    monkeypatch.delenv("TQ_JOIN_NO_FAST", raising=False)
    monkeypatch.setenv("TQ_JOIN_PART_ROWS", str(part_rows))


def _join(lib, bcols, pcols, jt=INNER_JOIN, oir=True, pkey=0):
    btypes, ptypes = [c.tp for c in bcols], [c.tp for c in pcols]
    e = HashJoinExec(MockDataSource(ptypes, pcols, 1 << 20), MockDataSource(btypes, bcols, 1 << 20), [pkey], [0], jt, oir)
    e.Open()
    got = e.drain()
    path = C.c_int32(-1)
    L.check(lib.tq_join_build_path(e.handle, C.byref(path)))
    e.Close()
    assert_same_multiset(got, O.hash_join(jt, oir, btypes, bcols, ptypes, pcols, [0], [pkey]))
    return path.value


def _build_cols(bk, nb):
    with np.errstate(over="ignore"):
        return [Column(INT64, bk)] + [Column(INT64, bk * (c + 3) + c) for c in range(1, nb)]


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("nb", [1, 2, 3, 4])
def test_cta_build_positional_probe(lib, monkeypatch, shape, nb):
    """16-byte (1-2 build columns) and 32-byte (3-4) entries, one or several sub-tables per slab; some probe keys miss"""
    n, part_rows = SHAPES[shape]
    g = cta_geometry(n, nb, part_rows)
    assert g is not None and (g["lbits"] == 0) == (shape == "one_per_slab")
    _switches(monkeypatch, part_rows)
    rng = np.random.default_rng(nb * 11 + len(shape))
    bk = rng.permutation(n * 5 // 4)[:n].astype(np.int64)
    npr = 2_000_000
    pk = rng.integers(0, n * 5 // 4, npr).astype(np.int64)
    path = _join(lib, _build_cols(bk, nb), [Column(INT64, pk), Column(FLOAT64, rng.random(npr))])
    assert path == L.TQ_JOIN_BUILD_CTA


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("jt,oir", [(LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True), (INNER_JOIN, True)])
def test_cta_build_general_probe(lib, monkeypatch, shape, jt, oir):
    """a CTA-built table probed by the general partitioned kernels: outer joins, and a nullable probe key column"""
    n, part_rows = SHAPES[shape]
    _switches(monkeypatch, part_rows)
    rng = np.random.default_rng(71 + jt + len(shape))
    bk = rng.permutation(n * 2)[:n].astype(np.int64)
    npr = 1_500_000
    pk = rng.integers(0, n * 2, npr).astype(np.int64)
    pcols = [Column(INT64, pk, rng.random(npr) > 0.05), Column(INT64, np.arange(npr))]
    assert _join(lib, _build_cols(bk, 2), pcols, jt, oir) == L.TQ_JOIN_BUILD_CTA


@pytest.mark.parametrize("nb,case", [(3, "unique"), (4, "unique"), (3, "duplicate")])
def test_cluster_build_where_no_cta_sub_table_fits(lib, monkeypatch, nb, case):
    """1.2e7 build rows of 32-byte entries: a sub-table one CTA holds would need more than 2^PART_MAX_BITS sub-tables, so
    the cluster build runs (its row count sets the table's); a duplicate key still hands over to the general build"""
    n = 12_000_000
    assert cta_geometry(n, nb) is None and H.stream_geometry(n, nb) is not None
    _switches(monkeypatch, H.PART_TARGET_ROWS)
    rng = np.random.default_rng(5 + nb)
    bk = rng.permutation(n * 5 // 4)[:n].astype(np.int64)
    if case == "duplicate":
        bk[n // 2] = bk[17]
    npr = 1_000_000
    pk = rng.integers(0, n * 5 // 4, npr).astype(np.int64)
    pk[:50] = bk[17]
    path = _join(lib, _build_cols(bk, nb), [Column(INT64, pk), Column(INT64, np.arange(npr))])
    assert path == (L.TQ_JOIN_BUILD_CLUSTER if case == "unique" else L.TQ_JOIN_BUILD_GENERAL)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("case", ["duplicate", "empty_marker"])
def test_cta_build_hands_over_to_general_build(lib, monkeypatch, shape, case):
    """a duplicate build key, or a build key equal to the empty marker: the general build takes over, same result"""
    n, part_rows = SHAPES[shape]
    _switches(monkeypatch, part_rows)
    rng = np.random.default_rng(13 if case == "duplicate" else 14)
    bk = rng.permutation(n * 2)[:n].astype(np.int64)
    if case == "duplicate":
        bk[n // 2] = bk[17]
    else:
        bk[n // 3] = EMPTY_MARKER
    npr = 1_000_000
    pk = rng.integers(0, n * 2, npr).astype(np.int64)
    pk[:50] = bk[17] if case == "duplicate" else EMPTY_MARKER
    path = _join(lib, [Column(INT64, bk), Column(INT64, np.arange(n))], [Column(INT64, pk), Column(INT64, np.arange(npr))])
    assert path == L.TQ_JOIN_BUILD_GENERAL


def _aimed(rng, counts, tbits, n, avoid):
    """counts[t] keys in sub-table t (exactly), the rest (n - sum) random in the other sub-tables"""
    parts = [H.join_keys(rng, c, t, tbits, 0, 1 << 32) for t, c in counts.items()]
    taken = np.concatenate(parts)
    rest = H.join_keys_not_in_tables(rng, n - len(taken), list(counts) + list(avoid), tbits, exclude=taken)
    bk = np.concatenate(parts + [rest])
    rng.shuffle(bk)
    return bk


@pytest.mark.parametrize("shape", list(SHAPES))
def test_cta_build_load_limit_hands_over(lib, monkeypatch, shape):
    """one sub-table gets ~1.45x its mean rows (over max_rows, under its capacity, inside its slab): flag 4 hands the build
    over; probed with hits and misses aimed at that sub-table"""
    n, part_rows = SHAPES[shape]
    g = cta_geometry(n, 2, part_rows)
    _switches(monkeypatch, part_rows)
    rng = np.random.default_rng(23 + len(shape))
    last = (1 << g["tbits"]) - 1
    n_hot = int(1.45 * n / (1 << g["tbits"]))
    assert n_hot >= 1.1 * g["max_rows"] and 1.1 * n_hot <= g["cap"]
    bk = _aimed(rng, {last: n_hot}, g["tbits"], n, [])
    cnt = np.bincount(H.table_of(H.hash_key(bk), g["tbits"]).astype(np.int64), minlength=last + 1)
    assert cnt[last] == n_hot and cnt[:last].max() < g["max_rows"]
    bins = np.bincount(H.table_of(H.hash_key(bk), g["bbits"]).astype(np.int64))
    assert bins.max() < g["bin_slab"]  # no slab overflows: the load limit alone hands over
    hot = bk[H.table_of(H.hash_key(bk), g["tbits"]) == np.uint64(last)]
    misses = H.join_keys(rng, 20000, last, g["tbits"], 0, 1 << 32, exclude=bk)
    pk = np.concatenate([hot, misses, rng.choice(bk, 400_000)])
    rng.shuffle(pk)
    path = _join(lib, _build_cols(bk, 2), [Column(INT64, pk), Column(INT64, np.arange(len(pk)))])
    assert path == L.TQ_JOIN_BUILD_GENERAL


def test_cta_build_skewed_slabs_stay(lib, monkeypatch):
    """slab counts far from even but inside the limits — the first slab holds 100 rows, the last ~1.13x the mean (each of
    its sub-tables just under max_rows) — and the CTA build keeps the table"""
    n, part_rows = SHAPES["several_per_slab"]
    g = cta_geometry(n, 2, part_rows)
    _switches(monkeypatch, part_rows)
    rng = np.random.default_rng(29)
    n_sub, n_sub_all = 1 << g["lbits"], 1 << g["tbits"]
    first = list(range(1, n_sub))                       # sub-tables of slab 0 other than sub-table 0: empty
    full = g["max_rows"] - 76
    counts = {0: 100, **{t: full for t in range(n_sub_all - n_sub, n_sub_all)}}
    bk = _aimed(rng, counts, g["tbits"], n, first)
    cnt = np.bincount(H.table_of(H.hash_key(bk), g["tbits"]).astype(np.int64), minlength=n_sub_all)
    assert cnt.max() <= g["max_rows"] and cnt[1:n_sub].sum() == 0
    bins = np.bincount(H.table_of(H.hash_key(bk), g["bbits"]).astype(np.int64))
    assert bins[0] == 100 and bins[-1] == n_sub * full and bins[-1] >= 1.1 * n / len(bins) and bins.max() < g["bin_slab"]
    npr = 1_000_000
    pk = np.concatenate([bk[:1000], rng.choice(bk, npr), rng.integers(0, 1 << 62, 20000)])
    path = _join(lib, _build_cols(bk, 2), [Column(INT64, pk), Column(INT64, np.arange(len(pk)))])
    assert path == L.TQ_JOIN_BUILD_CTA


@pytest.mark.parametrize("shape", list(SHAPES))
def test_cta_build_scatter_slab_overflow_hands_over(lib, monkeypatch, shape):
    """k_scatter_aos of the build side: one bin receives 1.3x slab_rows(n, n_bins) rows, so its slab overflows (cursor 2)
    and the rows past the slab's end are never inserted; the general build answers, with every row.  A full slab always
    holds more rows than its sub-tables may at the load limit (asserted below), so the build kernel also raises flag 4:
    no input overflows a slab while every sub-table stays within max_rows."""
    n, part_rows = SHAPES[shape]
    g = cta_geometry(n, 2, part_rows)
    assert g["bin_slab"] > (1 << g["lbits"]) * g["max_rows"]
    _switches(monkeypatch, part_rows)
    rng = np.random.default_rng(37 + len(shape))
    last = (1 << g["bbits"]) - 1
    n_hot = int(1.3 * g["bin_slab"])
    bk = _aimed(rng, {last: n_hot}, g["bbits"], n, [])
    bins = np.bincount(H.table_of(H.hash_key(bk), g["bbits"]).astype(np.int64), minlength=last + 1)
    assert bins[last] == n_hot and bins[:last].max() < g["bin_slab"]  # only the aimed slab overflows
    hot = bk[H.table_of(H.hash_key(bk), g["bbits"]) == np.uint64(last)]
    misses = H.join_keys(rng, 20000, last, g["bbits"], 0, 1 << 32, exclude=bk)
    pk = np.concatenate([hot, misses, rng.choice(bk, 400_000)])
    rng.shuffle(pk)
    path = _join(lib, _build_cols(bk, 2), [Column(INT64, pk), Column(INT64, np.arange(len(pk)))])
    assert path == L.TQ_JOIN_BUILD_GENERAL
