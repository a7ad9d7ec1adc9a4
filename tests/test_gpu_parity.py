"""GPU parity: the CUDA path (through the C-ABI) against the CPU oracle on the same seeded inputs.
Bit-exact for integer / key / COUNT work; SUM/AVG(float64) within 1e-9 relative (north_star)."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_py as O
from tinysql_b200 import _lib as L
from tinysql_b200 import expression as E
from tinysql_b200.chunk import FLOAT64, INT64, UINT64, Chunk, Column
from tinysql_b200.executor import (AGG_AVG, AGG_COUNT, AGG_FIRSTROW, AGG_MAX, AGG_MIN, AGG_SUM, INNER_JOIN, LEFT_OUTER_JOIN,
                                   RIGHT_OUTER_JOIN, HashAggExec, HashJoinExec, MockDataSource)
from util import assert_col_equal, assert_same_multiset, assert_same_ordered, gen_col

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 63, 64, 65, 1024, 4097, 100003]


# ------------------------------------------------------------------ vectorized builtins
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("ta,tb", [(INT64, INT64), (UINT64, UINT64), (UINT64, INT64), (INT64, UINT64)])
def test_compare_int(lib, n, ta, tb):
    rng = np.random.default_rng(n * 7 + ta * 3 + tb)
    a, b = gen_col(rng, ta, n), gen_col(rng, tb, n)
    if n > 10:  # force ties
        b.values[: n // 4] = a.values[: n // 4].astype(b.values.dtype)
    for op in range(6):
        rc, want = O.vec_compare_int(op, a, b)
        assert rc == 0
        assert_col_equal(E.vec_compare_int(op, a, b), want)


@pytest.mark.parametrize("n", [0, 65, 4097])
def test_compare_real(lib, n):
    rng = np.random.default_rng(n)
    a, b = gen_col(rng, FLOAT64, n), gen_col(rng, FLOAT64, n)
    if n > 10:
        b.values[:10] = a.values[:10]
        a.values[10] = np.nan
    for op in range(6):
        rc, want = O.vec_compare_real(op, a, b)
        assert_col_equal(E.vec_compare_real(op, a, b), want)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("op", [E.PLUS, E.MINUS, E.MUL])
@pytest.mark.parametrize("ta,tb", [(INT64, INT64), (UINT64, UINT64), (UINT64, INT64), (INT64, UINT64)])
def test_arith_int_no_overflow(lib, n, op, ta, tb):
    rng = np.random.default_rng(n + op * 11 + ta + 5 * tb)
    lim = (1 << 30) if op == E.MUL else (1 << 61)
    a = gen_col(rng, ta, n, lo=(0 if ta == UINT64 else -lim), hi=lim)
    b = gen_col(rng, tb, n, lo=(0 if tb == UINT64 else -lim), hi=lim)
    rc, want = O.vec_arith_int(op, a, b)
    if rc == 0:
        assert_col_equal(E.vec_arith_int(op, a, b), want)
    else:  # e.g. unsigned minus going negative: same error kind
        with pytest.raises(L.TQError) as ei:
            E.vec_arith_int(op, a, b)
        assert ei.value.status == rc


def test_arith_int_overflow_errors(lib):
    big = (1 << 63) - 1
    cases = [
        (E.PLUS, INT64, INT64, [1, big], [1, 1]),
        (E.PLUS, INT64, INT64, [-2, -big - 1], [1, -1]),
        (E.MINUS, INT64, INT64, [0, -big - 1], [0, 1]),
        (E.MUL, INT64, INT64, [3, big], [3, 2]),
        (E.MUL, INT64, INT64, [-1], [-big - 1]),  # Go's wrapping quotient hides this one: NO error in the reference
        (E.MUL, INT64, INT64, [-big - 1], [-1]),
        (E.PLUS, UINT64, UINT64, [np.uint64(1 << 63)], [np.uint64(1 << 63)]),
        (E.MINUS, UINT64, UINT64, [1], [2]),
        (E.MUL, UINT64, UINT64, [np.uint64(1 << 33)], [np.uint64(1 << 33)]),
        (E.MINUS, UINT64, INT64, [1], [2]),
        (E.MINUS, INT64, UINT64, [-1], [np.uint64(1 << 63)]),
        (E.PLUS, INT64, UINT64, [-5], [3]),
        (E.PLUS, UINT64, INT64, [3], [-5]),
    ]
    for op, ta, tb, av, bv in cases:
        a, b = Column(ta, av), Column(tb, bv)
        rc, want = O.vec_arith_int(op, a, b)
        if rc == 0:
            assert_col_equal(E.vec_arith_int(op, a, b), want)
        else:
            with pytest.raises(L.TQError) as ei:
                E.vec_arith_int(op, a, b)
            assert ei.value.status == rc, (op, ta, tb, av, bv)
    # overflow on a NULL row is ignored (`if result.IsNull(i) continue`)
    a = Column(INT64, [big, 5], [False, True])
    b = Column(INT64, [big, 6], [True, True])
    out = E.vec_arith_int(E.PLUS, a, b)
    assert out.tolist() == [None, 11]


@pytest.mark.parametrize("n", [0, 65, 4097, 100003])
@pytest.mark.parametrize("op", [E.PLUS, E.MINUS, E.MUL, E.DIV])
def test_arith_real(lib, n, op):
    rng = np.random.default_rng(n + op)
    a, b = gen_col(rng, FLOAT64, n), gen_col(rng, FLOAT64, n)
    if n > 10:
        b.values[3] = 0.0
        b.values[5] = -0.0
    rc, want, dz = O.vec_arith_real(op, a, b)
    got, gdz = E.vec_arith_real(op, a, b)
    assert rc == 0 and gdz == dz
    assert_col_equal(got, want)


def test_arith_real_overflow(lib):
    a, b = Column(FLOAT64, [1e308]), Column(FLOAT64, [1e308])
    for op in (E.PLUS, E.MUL):
        with pytest.raises(L.TQError) as ei:
            E.vec_arith_real(op, a, b)
        assert ei.value.status == L.TQ_ERR_OVERFLOW_DOUBLE
    with pytest.raises(L.TQError):
        E.vec_arith_real(E.DIV, a, Column(FLOAT64, [1e-300]))


@pytest.mark.parametrize("n", [0, 63, 4097])
def test_logic_unary_control(lib, n):
    rng = np.random.default_rng(n + 99)
    a = gen_col(rng, INT64, n, lo=-1, hi=2)
    b = gen_col(rng, INT64, n, lo=-1, hi=2)
    c = gen_col(rng, INT64, n, lo=-5, hi=5)
    f = gen_col(rng, FLOAT64, n)
    if n > 4:
        f.values[2] = 0.0
    for op in (E.AND, E.OR):
        assert_col_equal(E.vec_logic(op, a, b), O.vec_logic(op, a, b)[1])
    for op, arg in ((E.NOT_INT, a), (E.NOT_REAL, f), (E.MINUS_INT, c), (E.MINUS_REAL, f), (E.ISNULL, a)):
        rc, want = O.vec_unary(op, arg)
        assert rc == 0
        assert_col_equal(E.vec_unary(op, arg), want)
    assert_col_equal(E.vec_if(a, b, c), O.vec_if(a, b, c)[1])
    assert_col_equal(E.vec_ifnull(a, c), O.vec_ifnull(a, c)[1])
    assert_col_equal(E.vec_if(a, f, f), O.vec_if(a, f, f)[1])
    lst = [gen_col(rng, INT64, n, lo=-5, hi=5), gen_col(rng, UINT64, n, lo=0, hi=5), gen_col(rng, INT64, n, lo=-5, hi=5, null_frac=0)]
    assert_col_equal(E.vec_in_int(c, lst), O.vec_in_int(c, lst)[1])
    assert np.array_equal(E.vectorized_filter(a), O.vec_filter_int(a))


def test_unary_minus_overflow(lib):
    with pytest.raises(L.TQError) as ei:
        E.vec_unary(E.MINUS_INT, Column(INT64, [1, -(1 << 63)]))
    assert ei.value.status == L.TQ_ERR_OVERFLOW_BIGINT
    with pytest.raises(L.TQError):
        E.vec_unary(E.MINUS_INT, Column(UINT64, [np.uint64((1 << 63) + 1)]))
    assert E.vec_unary(E.MINUS_INT, Column(UINT64, [np.uint64(1 << 63)])).raw()[0] == np.uint64(1 << 63)


@pytest.mark.parametrize("n", [65, 100003, (1 << 22) + 77])
def test_lt_plus_fused(lib, n):
    rng = np.random.default_rng(n)
    a, b = gen_col(rng, INT64, n), gen_col(rng, INT64, n)  # [-2^62, 2^62): builtin_arithmetic_vec_test.go:47-52
    lt, plus = E.vec_lt_plus_int(a, b)
    assert_col_equal(lt, O.vec_compare_int(E.LT, a, b)[1])
    assert_col_equal(plus, O.vec_arith_int(E.PLUS, a, b)[1])


# ------------------------------------------------------------------ hash join
def _run_join(btypes, bcols, ptypes, pcols, jt=INNER_JOIN, outer_is_right=False, selected=None, chunk=1024, batch=0, bkey=0, pkey=0):
    inner = MockDataSource(btypes, bcols, chunk)
    outer = MockDataSource(ptypes, pcols, chunk)
    filt = None
    if selected is not None:
        state = {"pos": 0}

        def filt(chk):
            lo = state["pos"]
            state["pos"] += chk.num_rows()
            return selected[lo:state["pos"]]
    e = HashJoinExec(outer, inner, [pkey], [bkey], jt, outer_is_right, filt, batch)
    e.Open()
    got = e.drain()
    e.Close()
    want = O.hash_join(jt, outer_is_right, btypes, bcols, ptypes, pcols, [bkey], [pkey], selected)
    return got, want


@pytest.mark.parametrize("nb,npr", [(0, 0), (0, 100), (100, 0), (1, 1), (1000, 5000), (5000, 100000)])
@pytest.mark.parametrize("jt,oir", [(INNER_JOIN, False), (INNER_JOIN, True), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)])
def test_join_random(lib, nb, npr, jt, oir):
    rng = np.random.default_rng(nb * 31 + npr + jt)
    ndv = max(nb // 3, 1)
    bcols = [gen_col(rng, INT64, nb, 0.05, 0, ndv * 2), gen_col(rng, INT64, nb, 0.1), gen_col(rng, FLOAT64, nb, 0.1)]
    pcols = [gen_col(rng, FLOAT64, npr, 0.1), gen_col(rng, INT64, npr, 0.05, 0, ndv * 2)]
    got, want = _run_join([INT64, INT64, FLOAT64], bcols, [FLOAT64, INT64], pcols, jt, oir, pkey=1)
    assert_same_multiset(got, want)
    assert_same_ordered(got, want)  # single probe batch: (probe row asc, build insertion asc) order is kept


def test_join_selected_and_batches(lib):
    rng = np.random.default_rng(5)
    nb, npr = 3000, 40000
    bcols = [gen_col(rng, INT64, nb, 0.05, 0, 1000), gen_col(rng, INT64, nb, 0)]
    pcols = [gen_col(rng, INT64, npr, 0.05, 0, 1500), gen_col(rng, INT64, npr, 0.3)]
    sel = (rng.random(npr) < 0.7).astype(np.uint8)
    for jt, oir in ((INNER_JOIN, True), (LEFT_OUTER_JOIN, False)):
        # small device batches (4096 rows) and ragged chunk sizes exercise the accumulate / re-slice path
        got, want = _run_join([INT64, INT64], bcols, [INT64, INT64], pcols, jt, oir, selected=sel, chunk=1000, batch=4096)
        assert_same_multiset(got, want)


@pytest.mark.parametrize("jt,oir", [(INNER_JOIN, True), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)])
def test_join_partitioned_path(lib, jt, oir):
    """build side >= 65536 rows: partition tables in shared memory (TMA bulk loads), radix-scattered probe side."""
    rng = np.random.default_rng(77 + jt)
    nb, npr = 300000, 1200000
    bcols = [gen_col(rng, INT64, nb, 0.02, 0, 250000), gen_col(rng, INT64, nb, 0.1), gen_col(rng, FLOAT64, nb, 0.1)]
    pcols = [gen_col(rng, INT64, npr, 0.1), gen_col(rng, INT64, npr, 0.03, 0, 400000)]
    sel = (rng.random(npr) < 0.8).astype(np.uint8)
    got, want = _run_join([INT64, INT64, FLOAT64], bcols, [INT64, INT64], pcols, jt, oir, selected=sel, pkey=1, batch=1 << 19)
    assert_same_multiset(got, want)


def test_join_partitioned_skewed_probe_overflows_slab(lib):
    """a hot probe key sends most rows to ONE partition: the optimistic (histogram-free) scatter overflows its slab,
    flags it, and the batch is re-run on the exact histogram path — same answer"""
    rng = np.random.default_rng(8)
    nb, npr = 300000, 1000000
    bk = rng.permutation(nb).astype(np.int64)
    b = [Column(INT64, bk), Column(INT64, bk + 5)]
    pk = rng.integers(0, nb, npr).astype(np.int64)
    pk[rng.random(npr) < 0.8] = 4242
    p = [Column(INT64, pk), Column(INT64, np.arange(npr))]
    got, want = _run_join([INT64, INT64], b, [INT64, INT64], p, INNER_JOIN, True, chunk=1 << 20)
    assert_same_multiset(got, want)
    # second batch on the same handle takes the exact path from the start
    got, want = _run_join([INT64, INT64], b, [INT64, INT64], p, LEFT_OUTER_JOIN, False, chunk=1 << 18, batch=1 << 19)
    assert_same_multiset(got, want)


def test_join_partitioned_smem_tables(lib, monkeypatch):
    """~2400 build rows per partition: every partition table is TMA-bulk-loaded into shared memory"""
    monkeypatch.setenv("TQ_JOIN_PART_ROWS", "2400")
    rng = np.random.default_rng(123)
    nb, npr = 300000, 900000
    bcols = [gen_col(rng, INT64, nb, 0.02, 0, 200000), gen_col(rng, INT64, nb, 0.1)]
    pcols = [gen_col(rng, INT64, npr, 0.05, 0, 260000), gen_col(rng, FLOAT64, npr, 0.1)]
    for jt, oir in ((INNER_JOIN, False), (LEFT_OUTER_JOIN, False)):
        got, want = _run_join([INT64, INT64], bcols, [INT64, FLOAT64], pcols, jt, oir, batch=1 << 19)
        assert_same_multiset(got, want)


@pytest.mark.parametrize("no_fast", ["0", "1"])
def test_join_partitioned_unique_pk_fk(lib, monkeypatch, no_fast):
    """the C3 shape at 1/20 scale: unique build keys, every probe row matches exactly once
    (no_fast=0: the streaming build and the positional probe k_probe_pos; 1: the general build and the generic unique-key
    kernel)"""
    monkeypatch.setenv("TQ_JOIN_NO_FAST", no_fast)
    rng = np.random.default_rng(3)
    nb, npr = 500000, 5000000
    bk = rng.permutation(nb).astype(np.int64)
    b = [Column(INT64, bk), Column(INT64, bk * 7 + 1)]
    pk = rng.integers(0, nb, npr)
    p = [Column(INT64, pk), Column(INT64, np.arange(npr))]
    inner, outer = MockDataSource([INT64, INT64], b, 1 << 20), MockDataSource([INT64, INT64], p, 1 << 20)
    e = HashJoinExec(outer, inner, [0], [0], INNER_JOIN, True)
    e.Open()
    got = e.drain()
    e.Close()
    assert got.num_rows() == npr
    # size-independent properties: B.k == P.k, B.v == 7k+1, every probe row id appears exactly once
    assert np.array_equal(got.cols[0].values, got.cols[2].values)
    assert np.array_equal(got.cols[1].values, got.cols[0].values * 7 + 1)
    ids = np.sort(got.cols[3].values)
    assert np.array_equal(ids, np.arange(npr))
    assert np.array_equal(got.cols[2].values, pk[got.cols[3].values])


@pytest.mark.parametrize("nbc,npc", [(1, 1), (3, 2), (4, 4), (2, 3)])
def test_join_fast_kernel_shapes(lib, nbc, npc):
    """the positional probe k_probe_pos across column counts (16- and 32-byte entries), incl. misses and the empty-marker key
    (a build row with that key hands the table over from the streaming build to the general build)"""
    rng = np.random.default_rng(nbc * 10 + npc)
    nb, npr = 400000, 1500000
    s = np.int64(np.uint64(0xA5C3F00DDEADBEEF).astype(np.int64))
    bk = rng.permutation(nb * 2)[:nb].astype(np.int64)
    bk[7] = s
    bcols = [Column(INT64, bk)] + [Column(INT64, bk * (c + 3) + c) for c in range(1, nbc)]
    pk = rng.integers(0, nb * 2, npr).astype(np.int64)
    pk[11] = s
    pcols = [Column(FLOAT64, rng.random(npr)) for _ in range(npc - 1)] + [Column(INT64, pk)]
    got, want = _run_join([INT64] * nbc, bcols, [FLOAT64] * (npc - 1) + [INT64], pcols, INNER_JOIN, True, pkey=npc - 1, chunk=1 << 20)
    assert_same_multiset(got, want)


@pytest.mark.parametrize("stable", [False, True])
def test_join_large_host_chunks_direct_upload(lib, stable):
    """build and probe sides arriving as LARGE host columns (>= 2^18 rows per chunk): the build data goes straight to HBM
    (no pinned staging copy; the device columns grow twice here), probe pieces stream from the caller's buffers; with
    TQ_JOIN_STABLE_INPUT the uploads are not awaited before the call returns"""
    rng = np.random.default_rng(19)
    nb, npr = 700000, 2000000
    bcols = [gen_col(rng, INT64, nb, 0.02, 0, 600000), gen_col(rng, INT64, nb, 0.1), gen_col(rng, FLOAT64, nb, 0.1)]
    pcols = [gen_col(rng, INT64, npr, 0.1), gen_col(rng, INT64, npr, 0.03, 0, 800000)]
    inner, outer = MockDataSource([INT64, INT64, FLOAT64], bcols, 1 << 18), MockDataSource([INT64, INT64], pcols, 1 << 19)
    e = HashJoinExec(outer, inner, [1], [0], LEFT_OUTER_JOIN, False, None, 1 << 19, max_chunk_size=1 << 18, stable_input=stable)
    e.Open()
    got = e.drain()
    e.Close()
    want = O.hash_join(LEFT_OUTER_JOIN, False, [INT64, INT64, FLOAT64], bcols, [INT64, INT64], pcols, [0], [1])
    assert_same_multiset(got, want)


def test_join_duplicates_large_segments(lib):
    # 100 x 100 duplicate join (join_test.go:175-182) and a >32-row duplicate segment (bitonic path)
    b = [Column(INT64, [7] * 100 + [8] * 3), Column(INT64, list(range(103)))]
    p = [Column(INT64, [7] * 100 + [9]), Column(INT64, list(range(101)))]
    got, want = _run_join([INT64, INT64], b, [INT64, INT64], p)
    assert got.num_rows() == 10000
    assert_same_ordered(got, want)
    rng = np.random.default_rng(1)
    nb = 20000
    b = [Column(INT64, rng.integers(0, 7, nb)), Column(INT64, np.arange(nb))]
    p = [Column(INT64, np.arange(10)), Column(INT64, np.arange(10))]
    got, want = _run_join([INT64, INT64], b, [INT64, INT64], p)
    assert_same_ordered(got, want)


def test_join_signed_unsigned_keys(lib):
    # util/codec/codec_test.go:735-769: uint64(1) == int64(1); uint64(2^64-1) != int64(-1)
    b = [Column(UINT64, np.array([1, (1 << 64) - 1, 5], dtype=np.uint64))]
    p = [Column(INT64, [1, -1, 5, 7])]
    got, want = _run_join([UINT64], b, [INT64], p)
    assert_same_ordered(got, want)
    assert got.num_rows() == 2
    # both unsigned: the big value matches itself
    p2 = [Column(UINT64, np.array([(1 << 64) - 1], dtype=np.uint64))]
    got, want = _run_join([UINT64], b, [UINT64], p2)
    assert got.num_rows() == 1
    # float keys: bit equality (+0.0 != -0.0; NaN == same NaN)
    bf = [Column(FLOAT64, [0.0, np.nan, 1.5])]
    pf = [Column(FLOAT64, [-0.0, np.nan, 1.5, 0.0])]
    got, want = _run_join([FLOAT64], bf, [FLOAT64], pf)
    assert_same_ordered(got, want)
    assert got.num_rows() == 3
    # int vs double keys never match (flags differ)
    got, want = _run_join([FLOAT64], bf, [INT64], [Column(INT64, [0, 1])], LEFT_OUTER_JOIN)
    assert_same_ordered(got, want)


def test_join_sentinel_key(lib):
    s = np.int64(np.uint64(0xA5C3F00DDEADBEEF).astype(np.int64))
    b = [Column(INT64, [s, 1, s]), Column(INT64, [10, 11, 12])]
    p = [Column(INT64, [s, 2, 1])]
    got, want = _run_join([INT64, INT64], b, [INT64], p)
    assert_same_ordered(got, want)
    assert got.num_rows() == 3


def test_join_early_close(lib):
    inner = MockDataSource([INT64], [Column(INT64, np.arange(5000))])
    outer = MockDataSource([INT64], [Column(INT64, np.arange(5000))])
    e = HashJoinExec(outer, inner, [0], [0])
    e.Open()
    c = e.Next(1)  # `limit 1` then Close (join_test.go:175-182)
    assert c.num_rows() == 1
    e.Close()
    e2 = HashJoinExec(outer, inner, [0], [0])
    e2.Open()
    e2.Close()  # Close straight after Open


# ------------------------------------------------------------------ hash aggregation
def _run_agg(types, cols, group_by, funcs, chunk=1024, est=0):
    src = MockDataSource(types, cols, chunk)
    e = HashAggExec(src, group_by, funcs, est)
    e.Open()
    got = e.drain()
    e.Close()
    return got


def _sorted_by_key(chunk, key_idx):
    n = chunk.num_rows()
    nn = chunk.cols[key_idx].not_null()
    raw = chunk.cols[key_idx].raw().copy()
    raw[~nn] = 0
    order = np.lexsort((raw, nn))
    return [Column(c.tp, c.values[order], c.not_null()[order]) for c in chunk.cols]


@pytest.mark.parametrize("n,ndv", [(0, 1), (1, 1), (5000, 10), (200000, 5000), (300000, 250000)])
def test_agg_group_by(lib, n, ndv):
    rng = np.random.default_rng(n + ndv)
    k = gen_col(rng, INT64, n, 0.05, 0, ndv)
    x = gen_col(rng, FLOAT64, n, 0.1)
    x.values[:] = np.abs(x.values)  # no cancellation: tolerance 1e-9 relative is on SUM of same-signed terms
    v = gen_col(rng, INT64, n, 0.1, -1000, 1000)
    u = gen_col(rng, UINT64, n, 0.1, 0, 1 << 40)
    types, cols = [INT64, FLOAT64, INT64, UINT64], [k, x, v, u]
    funcs = [(AGG_SUM, 1), (AGG_COUNT, -1), (AGG_FIRSTROW, 0), (AGG_COUNT, 1), (AGG_AVG, 1), (AGG_SUM, 2), (AGG_AVG, 2), (AGG_MAX, 2),
             (AGG_MIN, 2), (AGG_MAX, 1), (AGG_MIN, 1), (AGG_MAX, 3), (AGG_MIN, 3)]
    got = _run_agg(types, cols, [0], funcs, est=ndv)
    rc, want = O.hash_agg(types, cols, [0], funcs, 4)
    assert rc == 0
    assert got.num_rows() == want.num_rows()
    g, w = _sorted_by_key(got, 2), _sorted_by_key(want, 2)
    for i, (f, a) in enumerate(funcs):
        if types[a if a >= 0 else 0] == FLOAT64 and f in (AGG_SUM, AGG_AVG):
            assert np.array_equal(g[i].not_null(), w[i].not_null())
            m = g[i].not_null()
            assert np.allclose(g[i].values[m], w[i].values[m], rtol=1e-9, atol=0)
        else:
            assert_col_equal(g[i], w[i])


def test_agg_scalar_and_empty(lib):
    # aggregate_test.go:51-69: count on an empty table => 0 / sum => NULL; with GROUP BY => no rows
    e = Column(INT64, [])
    got = _run_agg([INT64], [e], [], [(AGG_COUNT, 0), (AGG_SUM, 0), (AGG_MAX, 0)])
    assert got.rows() == [(0, None, None)]
    got = _run_agg([INT64], [e], [0], [(AGG_COUNT, 0)])
    assert got.num_rows() == 0
    rng = np.random.default_rng(3)
    v = gen_col(rng, INT64, 70001, 0.2, -50, 50)
    f = Column(FLOAT64, np.abs(rng.normal(size=70001)), rng.random(70001) > 0.2)
    funcs = [(AGG_COUNT, -1), (AGG_COUNT, 0), (AGG_SUM, 0), (AGG_AVG, 0), (AGG_MAX, 0), (AGG_MIN, 0), (AGG_SUM, 1), (AGG_AVG, 1)]
    got = _run_agg([INT64, FLOAT64], [v, f], [], funcs)
    rc, want = O.hash_agg([INT64, FLOAT64], [v, f], [], funcs, 3)
    assert rc == 0 and got.num_rows() == 1
    for i in range(6):
        assert_col_equal(got.cols[i], want.cols[i])
    for i in (6, 7):
        assert np.allclose(got.cols[i].values, want.cols[i].values, rtol=1e-9)


def test_agg_int_sum_overflow(lib):
    big = (1 << 62)
    v = Column(INT64, [big, big, big])
    with pytest.raises(L.TQError) as ei:
        _run_agg([INT64], [v], [], [(AGG_SUM, 0)])
    assert ei.value.status == L.TQ_ERR_OVERFLOW_BIGINT
    assert O.hash_agg([INT64], [v], [], [(AGG_SUM, 0)])[0] == 3
    # in range once the negatives arrive: both agree when every prefix is in range
    v2 = Column(INT64, [big, -big, big, -big, 5])
    got = _run_agg([INT64], [v2], [], [(AGG_SUM, 0)])
    assert got.rows() == [(5,)]


def test_agg_not_null_columns_compact_state(lib):
    """TQ_TYPE_NOT_NULL on the argument columns drops the SUM/MAX/MIN 'seen' word (16-byte group records)"""
    rng = np.random.default_rng(21)
    n = 250000
    k = Column(INT64, rng.integers(0, 40000, n))
    x = Column(FLOAT64, np.floor(rng.random(n) * 4096) / 16)  # dyadic values: float sums exact in any order
    v = Column(INT64, rng.integers(-1000, 1000, n))
    funcs = [(AGG_SUM, 1), (AGG_COUNT, -1), (AGG_FIRSTROW, 0), (AGG_MAX, 2), (AGG_MIN, 1), (AGG_AVG, 2)]
    src = MockDataSource([INT64, FLOAT64, INT64], [k, x, v], 1 << 16)
    e = HashAggExec(src, [0], funcs, 40000, not_null_cols=(0, 1, 2))
    e.Open()
    got = e.drain()
    e.Close()
    rc, want = O.hash_agg([INT64, FLOAT64, INT64], [k, x, v], [0], funcs, 2)
    g, w = _sorted_by_key(got, 2), _sorted_by_key(want, 2)
    for a, b in zip(g, w):
        assert_col_equal(a, b)


@pytest.mark.parametrize("n,ndv,est,hot", [(1300000, 900, 900, 0), (1500000, 60000, 60000, 0), (1200000, 250000, 100, 0),
                                           (1400000, 40000, 40000, 0.7), (6000000, 5000, 0, 0)])
def test_agg_shared_memory_preaggregation(lib, monkeypatch, n, ndv, est, hot):
    """large NOT NULL batches take the scatter -> shared-memory pre-aggregation -> merge path (k_agg_preagg): one table per
    CTA (ndv 900), partitioned (ndv 60000), an estimate far too small (tables fill up -> general path), a hot key that
    overflows its slab (-> general path), and no estimate at all (first batch general, the next ones pre-aggregated)"""
    monkeypatch.setenv("TQ_AGG_PREAGG_PART", "1")  # the radix-partitioned variant is opt-in (slower than the general path today)
    rng = np.random.default_rng(n % 1000 + ndv)
    kv = rng.integers(0, ndv, n)
    if hot:
        kv[rng.random(n) < hot] = 7
    k = Column(INT64, kv)
    x = Column(FLOAT64, np.floor(rng.random(n) * 4096) / 16)   # dyadic: float sums exact in any order
    y = Column(FLOAT64, np.floor(rng.random(n) * 1024) / 4)
    types, cols = [INT64, FLOAT64, FLOAT64], [k, x, y]
    funcs = [(AGG_SUM, 1), (AGG_COUNT, -1), (AGG_FIRSTROW, 0), (AGG_AVG, 2), (AGG_COUNT, 1)]
    src = MockDataSource(types, cols, 1 << 19)
    e = HashAggExec(src, [0], funcs, est, not_null_cols=(0, 1, 2))
    e.Open()
    got = e.drain()
    e.Close()
    rc, want = O.hash_agg(types, cols, [0], funcs, 2)
    assert rc == 0
    g, w = _sorted_by_key(got, 2), _sorted_by_key(want, 2)
    for a, b in zip(g, w):
        assert_col_equal(a, b)


def test_agg_preaggregation_marker_key_and_device_batch(lib):
    """one device-resident batch (the bench shape) holding the table's empty-marker value as a key: the pre-aggregation
    gives up and the general path answers"""
    from tinysql_b200.chunk import DeviceColumn
    rng = np.random.default_rng(77)
    n = 1 << 21
    kv = rng.integers(0, 3000, n)
    kv[5] = np.int64(np.uint64(0xA5C3F00DDEADBEEF).astype(np.int64))
    xv = np.floor(rng.random(n) * 256) / 2
    for with_marker in (True, False):
        kk = kv.copy()
        if not with_marker:
            kk[5] = 1
        dk, dx = DeviceColumn.from_host(Column(INT64, kk)), DeviceColumn.from_host(Column(FLOAT64, xv))
        it, gb = (C.c_int32 * 2)(INT64 | 0x100, FLOAT64 | 0x100), (C.c_int32 * 1)(0)
        fl = [(AGG_SUM, 1), (AGG_COUNT, -1), (AGG_FIRSTROW, 0)]
        fa = (L.TQAggFunc * 3)(*[L.TQAggFunc(f, a) for f, a in fl])
        d = L.TQAggDesc(2, it, 1, gb, 3, fa, 3000)
        h = C.c_void_p()
        L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
        cols = (L.TQColumn * 2)(dk.tq(), dx.tq())
        cols[0].null_bitmap = None
        cols[1].null_bitmap = None
        L.check(lib.tq_agg_put(h, cols, L.TQ_MEM_DEVICE))
        L.check(lib.tq_agg_eof(h))
        res = [Column.empty(t, 4096) for t in (FLOAT64, INT64, INT64)]
        from tinysql_b200.chunk import tq_array
        nr, eof = C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_agg_next(h, 4096, tq_array(res, 4096), C.byref(nr), C.byref(eof)))
        L.check(lib.tq_agg_destroy(h))
        got = Chunk([Column(c.tp, c.values[: nr.value], c.not_null()[: nr.value]) for c in res])
        rc, want = O.hash_agg([INT64, FLOAT64], [Column(INT64, kk), Column(FLOAT64, xv)], [0], fl, 1)
        gs, ws = _sorted_by_key(got, 2), _sorted_by_key(want, 2)
        for a, b in zip(gs, ws):
            assert_col_equal(a, b)
        dk.free(); dx.free()


def test_agg_table_growth(lib):
    # est_groups far too small: the table grows several times and deferred rows are replayed
    rng = np.random.default_rng(9)
    n = 400000
    k = Column(INT64, rng.integers(0, 300000, n))
    x = Column(INT64, rng.integers(-100, 100, n))
    funcs = [(AGG_FIRSTROW, 0), (AGG_SUM, 1), (AGG_COUNT, -1)]
    got = _run_agg([INT64, INT64], [k, x], [0], funcs, est=1)
    rc, want = O.hash_agg([INT64, INT64], [k, x], [0], funcs)
    g, w = _sorted_by_key(got, 0), _sorted_by_key(want, 0)
    for a, b in zip(g, w):
        assert_col_equal(a, b)


# ------------------------------------------------------------------ multi-GPU shard boundary, exercised on ONE GPU
def test_partition_count_and_push_local(lib):
    """tq_partition_count_device + tq_partition_push_device with all destination buffers on this GPU: every row lands in
    the partition (mix64(key) >> 40) % n_parts, at the offsets the count pass implies, nothing lost or duplicated"""
    from tinysql_b200 import dist as D
    from tinysql_b200.chunk import DeviceColumn
    rng = np.random.default_rng(31)
    for n, n_parts in ((0, 2), (1, 2), (5000, 3), (300001, 4), (1200000, 8)):
        k = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
        v = np.arange(n, dtype=np.int64)
        dk, dv = DeviceColumn.from_host(Column(INT64, k)), DeviceColumn.from_host(Column(INT64, v))
        tk = dk.tq(); tk.null_bitmap = None
        counts = (C.c_int64 * n_parts)()
        L.check(lib.tq_partition_count_device(C.byref(tk), n, n_parts, counts))
        want_dest = D.dest_rank_np(k, n_parts) if n else np.zeros(0, np.int64)
        assert list(counts) == list(np.bincount(want_dest, minlength=n_parts))
        # destination q gets its own pair of buffers, with a 7-row offset to prove offsets are honoured
        bufs = [[DeviceColumn(INT64, int(counts[q]) + 7, with_bitmap=False) for _ in range(2)] for q in range(n_parts)]
        dest = (C.c_void_p * (n_parts * 2))()
        for q in range(n_parts):
            for c in range(2):
                dest[q * 2 + c] = bufs[q][c]._data.value
        offs = (C.c_int64 * n_parts)(*([7] * n_parts))
        cols = (L.TQColumn * 2)(dk.tq(), dv.tq())
        cols[0].null_bitmap = None
        cols[1].null_bitmap = None
        L.check(lib.tq_partition_push_device(2, cols, 0, n, n_parts, dest, offs))
        seen = []
        for q in range(n_parts):
            kq = bufs[q][0].to_host().values[7:]
            vq = bufs[q][1].to_host().values[7:]
            assert np.all(D.dest_rank_np(kq, n_parts) == q)
            assert np.array_equal(k[vq], kq)  # the payload still travels with its key
            seen.append(vq)
            for b in bufs[q]:
                b.free()
        allv = np.sort(np.concatenate(seen)) if seen else np.zeros(0, np.int64)
        assert np.array_equal(allv, np.arange(n))
        dk.free(); dv.free()


# ------------------------------------------------------------------ partial -> final aggregation (the multi-GPU agg shape)
def test_agg_partial_export_and_final_merge(lib):
    """two Partial1 handles over disjoint halves -> tq_agg_export_partial -> one Final handle via tq_agg_merge_partial
    == the oracle over all rows (AggFuncDesc.Split, descriptor.go:57-92; MergePartialResult semantics)"""
    from tinysql_b200.chunk import DeviceColumn, device_to_host, tq_array
    rng = np.random.default_rng(44)
    n = 120000
    k = gen_col(rng, INT64, n, 0.03, 0, 3000)
    x = gen_col(rng, FLOAT64, n, 0.1)
    x.values[:] = np.floor(np.abs(x.values)) / 4          # dyadic: float sums exact in any order
    v = gen_col(rng, INT64, n, 0.1, -500, 500)
    types = [INT64, FLOAT64, INT64]
    funcs = [(AGG_FIRSTROW, 0), (AGG_COUNT, -1), (AGG_COUNT, 2), (AGG_SUM, 1), (AGG_AVG, 1), (AGG_SUM, 2), (AGG_AVG, 2), (AGG_MAX, 2), (AGG_MIN, 1)]

    def make():
        it, gb = (C.c_int32 * 3)(*types), (C.c_int32 * 1)(0)
        fa = (L.TQAggFunc * len(funcs))(*[L.TQAggFunc(f, a) for f, a in funcs])
        d = L.TQAggDesc(3, it, 1, gb, len(funcs), fa, 3000)
        h = C.c_void_p()
        L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
        return h, (it, gb, fa)
    final, keep_f = make()
    width = C.c_int32(0)
    L.check(lib.tq_agg_partial_width(final, C.byref(width)))
    assert width.value == 1 + len(funcs) + 2               # key + one column per function, AVG twice (count, sum)
    for lo, hi in ((0, n // 2), (n // 2, n)):
        part, keep_p = make()
        cols = [c.slice(lo, hi) for c in (k, x, v)]
        L.check(lib.tq_agg_put(part, tq_array(cols), L.TQ_MEM_HOST))
        L.check(lib.tq_agg_eof(part))
        out = (L.TQColumn * width.value)()
        rows = C.c_int64(0)
        L.check(lib.tq_agg_export_partial(part, out, C.byref(rows)))   # device-resident partial rows
        assert rows.value > 0
        L.check(lib.tq_agg_merge_partial(final, out, L.TQ_MEM_DEVICE))
        L.check(lib.tq_agg_destroy(part))
    L.check(lib.tq_agg_eof(final))
    out_types = []
    for i in range(len(funcs)):
        t = C.c_int32(0)
        L.check(lib.tq_agg_output_type(final, i, C.byref(t)))
        out_types.append(t.value)
    res = [Column.empty(t, 4096) for t in out_types]
    got_cols = [[] for _ in funcs]
    got_nn = [[] for _ in funcs]
    while True:
        arr = tq_array(res, 4096)
        nr, eof = C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_agg_next(final, 4096, arr, C.byref(nr), C.byref(eof)))
        if nr.value == 0:
            break
        for i, c in enumerate(res):
            got_cols[i].append(c.values[: nr.value].copy())
            got_nn[i].append(c.not_null()[: nr.value].copy())
    L.check(lib.tq_agg_destroy(final))
    got = Chunk([Column(t, np.concatenate(a), np.concatenate(b)) for t, a, b in zip(out_types, got_cols, got_nn)])
    rc, want = O.hash_agg(types, [k, x, v], [0], funcs, 2)
    assert rc == 0 and got.num_rows() == want.num_rows()
    g, w = _sorted_by_key(got, 0), _sorted_by_key(want, 0)
    for a, b in zip(g, w):
        assert_col_equal(a, b)


def test_vec_builtins_device_memory_mode(lib):
    """TQ_MEM_DEVICE: operands and results stay in HBM (the path a fused Selection/Projection feeding the operators takes)"""
    from tinysql_b200.chunk import DeviceColumn
    rng = np.random.default_rng(2)
    for n in (1, 64, 100003):
        a, b = gen_col(rng, INT64, n, 0.2), gen_col(rng, INT64, n, 0.2)
        da, db = DeviceColumn.from_host(a), DeviceColumn.from_host(b)
        out1, out2 = DeviceColumn(INT64, n), DeviceColumn(INT64, n)
        ta, tb, t1, t2 = da.tq(), db.tq(), out1.tq(), out2.tq()
        L.check(lib.tq_vec_compare_int(E.GE, n, C.byref(ta), 0, C.byref(tb), 0, C.byref(t1), L.TQ_MEM_DEVICE))
        assert_col_equal(out1.to_host(), O.vec_compare_int(E.GE, a, b)[1])
        L.check(lib.tq_vec_lt_plus_int(n, C.byref(ta), C.byref(tb), C.byref(t1), C.byref(t2), L.TQ_MEM_DEVICE))
        assert_col_equal(out1.to_host(), O.vec_compare_int(E.LT, a, b)[1])
        assert_col_equal(out2.to_host(), O.vec_arith_int(E.PLUS, a, b)[1])
        sel = np.zeros(n, dtype=np.uint8)
        dsel = C.c_void_p()
        L.check(lib.tq_device_alloc(n, C.byref(dsel)))
        L.check(lib.tq_vec_filter_int(n, C.byref(ta), dsel, L.TQ_MEM_DEVICE))
        L.check(lib.tq_memcpy_d2h(sel.ctypes.data, dsel, n))
        assert np.array_equal(sel, O.vec_filter_int(a))
        lib.tq_device_free(dsel)
        for d in (da, db, out1, out2):
            d.free()


# ------------------------------------------------------------------ streaming PK-FK pipeline (join_stream.cuh)
@pytest.mark.parametrize("miss_factor", [1.0, 1.3, 3.0])
def test_join_stream_pipeline_holes(lib, miss_factor):
    """positional probe output + hole filling: no misses (only the 32-row padding of each partition), a moderate number of
    misses (device-driven fill) and a majority of misses (host-sized fill) — multiset against the oracle"""
    rng = np.random.default_rng(int(miss_factor * 10))
    nb, npr = 400000, 3000000
    bk = rng.permutation(int(nb * miss_factor))[:nb].astype(np.int64)
    pk = rng.integers(0, int(nb * miss_factor), npr).astype(np.int64)
    got, want = _run_join([INT64, INT64], [Column(INT64, bk), Column(INT64, bk * 3 + 1)], [INT64, INT64], [Column(INT64, pk), Column(INT64, np.arange(npr))],
                          INNER_JOIN, True, chunk=1 << 20)
    assert_same_multiset(got, want)


def test_join_stream_pipeline_outer_filter_and_sign_mix(lib):
    """outerSideFilter rows and keys that cannot match across signedness are dropped by the scatter"""
    rng = np.random.default_rng(77)
    nb, npr = 300000, 1000000
    bk = rng.permutation(nb).astype(np.int64)
    pk = rng.integers(-1000, nb, npr).astype(np.int64).astype(np.uint64)
    sel = (rng.random(npr) > 0.3).astype(np.uint8)
    got, want = _run_join([INT64, INT64], [Column(INT64, bk), Column(INT64, bk + 5)], [UINT64, FLOAT64], [Column(UINT64, pk), Column(FLOAT64, rng.random(npr))],
                          INNER_JOIN, False, selected=sel, chunk=1 << 19)
    assert_same_multiset(got, want)


def test_join_stream_pipeline_device_columns_unaligned(lib):
    """device-resident inputs whose pointers are only 8-byte aligned and whose row counts are odd: the scatter falls back
    from TMA bulk copies to plain loads; checked by size-independent properties"""
    from tinysql_b200.chunk import DeviceColumn
    rng = np.random.default_rng(5)
    nb, npr = 500001, 2000003
    bk = rng.permutation(nb).astype(np.int64)
    pk = rng.integers(0, nb, npr).astype(np.int64)
    for shift_rows in (0, 1):
        d_b = [DeviceColumn.from_host(Column(INT64, np.concatenate([[0] * shift_rows, x]))) for x in (bk, bk * 7 + 1)]
        d_p = [DeviceColumn.from_host(Column(INT64, np.concatenate([[0] * shift_rows, x]))) for x in (pk, np.arange(npr))]
        t = (C.c_int32 * 2)(1, 1)
        k = (C.c_int32 * 1)(0)
        d = L.TQJoinDesc(0, 1, 2, t, 2, t, 1, k, k, 0, 0)
        h = C.c_void_p()
        L.check(lib.tq_join_create(C.byref(d), C.byref(h)))

        def arr(cols, n):
            a = (L.TQColumn * 2)()
            for i, c in enumerate(cols):
                a[i].length, a[i].data, a[i].null_bitmap, a[i].offsets = n, c._data.value + 8 * shift_rows, None, None
            return a
        L.check(lib.tq_join_put_build(h, arr(d_b, nb), L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        L.check(lib.tq_join_put_probe(h, arr(d_p, npr), None, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_probe_eof(h))
        out = (L.TQColumn * 4)()
        n, eof = C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
        assert n.value == npr
        from tinysql_b200.chunk import device_to_host
        cols = [device_to_host(INT64, out[c].data, None, npr).values for c in range(4)]
        L.check(lib.tq_join_destroy(h))
        assert np.array_equal(cols[0], cols[2]) and np.array_equal(cols[1], cols[0] * 7 + 1)
        assert np.array_equal(np.sort(cols[3]), np.arange(npr)) and np.array_equal(cols[2], pk[cols[3]])
        for c in d_b + d_p:
            c.free()


@pytest.mark.parametrize("n,ndv,est", [(3, 2, 0), (200000, 50000, 60000), (700000, 300000, 1)])
def test_agg_fast_update_path(lib, n, ndv, est):
    """k_agg_update_fast: NOT NULL integer GROUP BY column, COUNT(*) + COUNT(col) + SUM(double NOT NULL) x 2 + FIRSTROW(key); with table
    growth (est far too small: deferred rows are replayed by the generic kernel into the same table) and the empty-marker key"""
    rng = np.random.default_rng(n)
    kv = rng.integers(-ndv // 2, ndv // 2 + 1, n)
    kv[0] = np.int64(np.uint64(0xA5C3F00DDEADBEEF).astype(np.int64))
    k = Column(UINT64 if n == 3 else INT64, kv)
    x = Column(FLOAT64, np.floor(rng.random(n) * 4096) / 16)   # dyadic values: float sums exact in any order
    y = Column(FLOAT64, np.floor(rng.random(n) * 1024) / 4)
    tp = [k.tp, FLOAT64, FLOAT64]
    funcs = [(AGG_SUM, 1), (AGG_COUNT, -1), (AGG_FIRSTROW, 0), (AGG_SUM, 2), (AGG_COUNT, 2)]
    src = MockDataSource(tp, [k, x, y], 1 << 16)
    e = HashAggExec(src, [0], funcs, est, not_null_cols=(0, 1, 2))
    e.Open()
    got = e.drain()
    e.Close()
    rc, want = O.hash_agg(tp, [k, x, y], [0], funcs, 2)
    assert rc == 0
    g, w = _sorted_by_key(got, 2), _sorted_by_key(want, 2)
    for a, b in zip(g, w):
        assert_col_equal(a, b)
