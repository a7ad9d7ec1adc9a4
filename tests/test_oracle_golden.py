"""CPU suite, part 1: the oracle (oracle/oracle.c) pinned against the known-answer tests the reference's own
test-suite holds for this path, re-expressed (the Go tests cannot run here: no Go toolchain, hot functions
are course stubs).  Each case cites the reference test it restates (paths relative to the reference repository)."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O
from tinysql_b200.chunk import FLOAT64, INT64, UINT64, Chunk, Column

INNER, LEFT, RIGHT = 0, 1, 2
COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)
N = None


def icol(vals, tp=INT64):
    nn = [v is not None for v in vals]
    return Column(tp, [0 if v is None else v for v in vals], nn)


def table(rows, ncols=None):
    ncols = ncols if ncols is not None else (len(rows[0]) if rows else 0)
    return [icol([r[c] for r in rows]) for c in range(ncols)]


def join(lhs_rows, rhs_rows, lkey, rkey, jt, inner_is_left, ncl=None, ncr=None):
    """lhs/rhs as in the SQL text; returns output rows (lhs cols ++ rhs cols) in oracle order."""
    l, r = table(lhs_rows, ncl), table(rhs_rows, ncr)
    if inner_is_left:
        out = O.hash_join(jt, True, [INT64] * len(l), l, [INT64] * len(r), r, [lkey], [rkey])
    else:
        out = O.hash_join(jt, False, [INT64] * len(r), r, [INT64] * len(l), l, [rkey], [lkey])
    return out.rows()


# ------------------------------------------------------------------ hash/fnv + codec
def fnv1_64(data):
    h = 14695981039346656037
    for b in data:
        h = (h * 1099511628211) & 0xFFFFFFFFFFFFFFFF
        h ^= b
    return h


def test_fnv1_known_answer():
    # Go hash/fnv golden64 vector for New64(): FNV-1("a") = af63bd4c8601b7be
    assert fnv1_64(b"a") == 0xAF63BD4C8601B7BE
    assert fnv1_64(b"") == 0xCBF29CE484222325


def _hash(cols, types, keys, row):
    hn = C.c_int(0)
    from tinysql_b200.chunk import tq_array
    h = O.load().orc_hash_row(C.c_int(len(keys)), (C.c_int * len(types))(*types), tq_array(cols), (C.c_int * len(keys))(*keys), C.c_int64(row), C.byref(hn))
    return h, hn.value


def test_hash_row_is_fnv1_of_flag_and_raw_bytes():
    # executor/hash_table.go:55-72 + util/codec/codec.go:249-276: h.Write(flag); h.Write(8 raw little-endian bytes)
    col = icol([1, -5, N, 123456789012])
    for row, v in enumerate([1, -5, None, 123456789012]):
        h, hn = _hash([col], [INT64], [0], row)
        if v is None:
            assert hn == 1 and h == fnv1_64(bytes([0]))  # NilFlag only
        else:
            assert hn == 0 and h == fnv1_64(bytes([8]) + int(v).to_bytes(8, "little", signed=True))
    f = Column(FLOAT64, [1.5])
    assert _hash([f], [FLOAT64], [0], 0)[0] == fnv1_64(bytes([5]) + np.float64(1.5).tobytes())


def test_hash_chunk_row_equalities():
    # util/codec/codec_test.go:735-769 TestHashChunkRow: uint64(1) == int64(1); uint64(MaxUint64) != int64(-1)
    u = Column(UINT64, np.array([1, (1 << 64) - 1], dtype=np.uint64))
    i = Column(INT64, [1, -1])
    assert _hash([u], [UINT64], [0], 0)[0] == _hash([i], [INT64], [0], 0)[0]
    assert _hash([u], [UINT64], [0], 1)[0] != _hash([i], [INT64], [0], 1)[0]
    from tinysql_b200.chunk import tq_array
    lib = O.load()
    eq = lambda r1, r2: lib.orc_equal_row(C.c_int(1), (C.c_int * 1)(UINT64), tq_array([u]), (C.c_int * 1)(0), C.c_int64(r1),
                                          (C.c_int * 1)(INT64), tq_array([i]), (C.c_int * 1)(0), C.c_int64(r2))
    assert eq(0, 0) == 1 and eq(1, 1) == 0


def test_hash_chunk_columns_vector_equals_row_and_flags_null():
    # util/codec/codec_test.go:811-866 TestHashChunkColumns: multi-column vector hash == row hash; NULL flagged
    a, b = icol([1, N, 3]), Column(FLOAT64, [0.5, 1.5, 2.5], [True, True, False])
    for row in range(3):
        h, hn = _hash([a, b], [INT64, FLOAT64], [0, 1], row)
        data = b""
        exp_null = 0
        for col, flag in ((a, 8), (b, 5)):
            if col.not_null()[row]:
                data += bytes([flag]) + col.values[row].tobytes()
            else:
                data += bytes([0])
                exp_null = 1
        assert (h, hn) == (fnv1_64(data), exp_null)


def test_row_hash_map():
    # executor/hash_table_test.go:21-50 TestRowHashMap: insertion-order Get across entry-slab growth, Len
    lib = O.load()
    lib.orc_rowmap_put.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32]
    lib.orc_rowmap_get.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_int64]
    lib.orc_rowmap_len.argtypes = [C.c_void_p]
    lib.orc_rowmap_free.argtypes = [C.c_void_p]
    m = lib.orc_rowmap_new()
    lib.orc_rowmap_put(m, 1, 1, 1)
    buf = (C.c_uint32 * 2)()
    assert lib.orc_rowmap_get(m, 1, buf, 1) == 1 and list(buf) == [1, 1]
    lib.orc_rowmap_free(m)
    slab = 64  # initialEntrySliceLen (hash_table.go:178)
    raw = {i: [(i, j) for j in range(slab * i)] for i in range(10)}
    m = lib.orc_rowmap_new()
    for j in range(slab * 9):
        for i in range(9, -1, -1):
            if not j < slab * i:
                break
            lib.orc_rowmap_put(m, i, raw[i][j][0], raw[i][j][1])
    total = 0
    for i in range(10):
        total += len(raw[i])
        buf = (C.c_uint32 * (2 * max(len(raw[i]), 1)))()
        assert lib.orc_rowmap_get(m, i, buf, len(raw[i])) == len(raw[i])
        assert [(buf[2 * k], buf[2 * k + 1]) for k in range(len(raw[i]))] == raw[i]
    assert lib.orc_rowmap_len(m) == total
    lib.orc_rowmap_free(m)


# ------------------------------------------------------------------ executor/join_test.go TestJoin (:36-150)
def test_join_left_right_outer_goldens():
    t, t1 = [(1, 1), (2, 2)], [(2, 3), (4, 4)]
    # select * from t left outer join t1 on t.c1 = t1.c1  [then: where t.c1 = 1 or t1.c2 > 20]  (:72-75)
    rows = join(t, t1, 0, 0, LEFT, inner_is_left=False)
    assert rows == [(1, 1, N, N), (2, 2, 2, 3)]
    assert [r for r in rows if r[0] == 1 or (r[3] is not None and r[3] > 20)] == [(1, 1, N, N)]
    # select * from t1 right outer join t on t.c1 = t1.c1 where ...  -> "<nil> <nil> 1 1"  (:76-77)
    rows = join(t1, t, 0, 0, RIGHT, inner_is_left=True)
    assert [r for r in rows if r[2] == 1 or (r[1] is not None and r[1] > 20)] == [(N, N, 1, 1)]
    # select * from t right outer join t1 ... where t.c1 = 1 or t1.c2 > 20 -> empty  (:78-79)
    rows = join(t, t1, 0, 0, RIGHT, inner_is_left=True)
    assert rows == [(2, 2, 2, 3), (N, N, 4, 4)]
    assert [r for r in rows if r[0] == 1 or (r[3] is not None and r[3] > 20)] == []
    # left outer join ... where t1.c1 = 3 or false -> empty  (:80-81)
    assert [r for r in join(t, t1, 0, 0, LEFT, False) if r[2] == 3] == []


def test_join_outer_filter_is_a_miss():
    # select * from t left outer join t1 on t.c1 = t1.c1 and t.c1 != 1 order by t1.c1 -> "1 1 <nil> <nil>","2 2 2 3" (:82-83)
    # `t.c1 != 1` is an outer-side condition: it arrives as outerSideFilter / selected[] (join.go:328,344)
    t, t1 = table([(1, 1), (2, 2)]), table([(2, 3), (4, 4)])
    sel = np.array([0, 1], dtype=np.uint8)
    out = O.hash_join(LEFT, False, [INT64, INT64], t1, [INT64, INT64], t, [0], [0], sel)
    assert out.rows() == [(1, 1, N, N), (2, 2, 2, 3)]


def test_join_three_tables():
    # t1 left join t2 on t1.c1=t2.c1 right join t3 on t2.c1=t3.c1 order by ... (:97-98)
    t1, t2, t3 = [(1, 1), (2, 2), (3, 3)], [(1, 1), (3, 3), (5, 5)], [(1, 1), (5, 5), (9, 9)]
    a = join(t1, t2, 0, 0, LEFT, False)
    assert a == [(1, 1, 1, 1), (2, 2, N, N), (3, 3, 3, 3)]
    b = join(a, t3, 2, 0, RIGHT, True, ncl=4)
    key = lambda r: tuple((0, 0) if v is None else (1, v) for v in r)
    assert sorted(b, key=key) == [(N, N, N, N, 5, 5), (N, N, N, N, 9, 9), (1, 1, 1, 1, 1, 1)]


def test_join_duplicates_and_order():
    # 3 x 3 duplicate self join -> nine "1 1" rows (:100-104)
    t1 = [(1,), (1,), (1,)]
    assert join(t1, t1, 0, 0, INNER, False) == [(1, 1)] * 9
    # a.c1 = b.c1 over 1..7 (:111-113) and `a.c1 + b.c1 > 5` as a post-filter (:115-116)
    t = [(i,) for i in range(1, 8)]
    rows = join(t, t, 0, 0, INNER, False)
    assert [r[0] for r in rows] == [1, 2, 3, 4, 5, 6, 7]
    assert [r[0] for r in rows if r[0] + r[1] > 5] == [3, 4, 5, 6, 7]
    # t join t1 on t.a = t1.a -> "1 1 1 2","1 1 1 3","1 1 1 4","3 3 3 4" in THIS order (no .Sort(), :134-136):
    # probe row order, matches in build insertion order
    t, t1 = [(1, 1), (2, 2), (3, 3)], [(1, 2), (1, 3), (1, 4), (3, 4), (4, 5)]
    assert join(t, t1, 0, 0, INNER, False) == [(1, 1, 1, 2), (1, 1, 1, 3), (1, 1, 1, 4), (3, 3, 3, 4)]
    # t right outer join t1 on t.a = t1.a -> ... "<nil> <nil> 4 5" (:144-146)
    assert join(t, t1, 0, 0, RIGHT, True) == [(1, 1, 1, 2), (1, 1, 1, 3), (1, 1, 1, 4), (3, 3, 3, 4), (N, N, 4, 5)]
    # t1 join t on t.a = t1.a and t.a < t1.b (:137-139): other condition applied on the joined rows
    rows = join(t1, t, 0, 0, INNER, False)
    assert [r for r in rows if r[2] < r[1]] == [(1, 2, 1, 1), (1, 3, 1, 1), (1, 4, 1, 1), (3, 4, 3, 3)]


def test_join_null_keys_never_match():
    # hash_table.go:161-163 (build rows with NULL keys are not inserted); join.go:344 (probe NULL key -> miss)
    b, p = [(N, 1), (1, 2)], [(N, 10), (1, 11)]
    assert join(p, b, 0, 0, INNER, False) == [(1, 11, 1, 2)]
    assert join(p, b, 0, 0, LEFT, False) == [(N, 10, N, N), (1, 11, 1, 2)]


# ------------------------------------------------------------------ aggfuncs known answers
def agg(vals, tp, funcs, group=None, workers=1):
    cols = [Column(tp, [0 if v is None else v for v in vals], [v is not None for v in vals])]
    types = [tp]
    gb = []
    if group is not None:
        cols.append(icol(group))
        types.append(INT64)
        gb = [1]
    rc, out = O.hash_agg(types, cols, gb, funcs, workers)
    return rc, out.rows()


@pytest.mark.parametrize("tp,conv", [(INT64, int), (FLOAT64, float)])
def test_sum_avg_count_goldens(tp, conv):
    data = [conv(i) for i in range(5)]            # getDataGenFunc: row i -> i (aggfunc_test.go:152-166)
    # func_sum_test.go TestSum: empty -> NULL, 0..4 -> 10;  func_avg_test.go TestAvg: -> 2.0;  func_count_test.go: 0 -> 5
    assert agg([], tp, [(SUM, 0), (AVG, 0), (COUNT, 0)]) == (0, [(N, N, 0)])
    rc, rows = agg(data, tp, [(SUM, 0), (AVG, 0), (COUNT, 0)])
    assert rc == 0 and rows == [(conv(10), conv(2), 5)]
    # TestMergePartialResult4Sum / 4Avg: partial over rows 0..4 (10 / 2.0) merged with partial over rows 2..4 (9 / 3.0)
    # -> 19 and 19/8: 2.375 for DOUBLE, truncating 2 for BIGINT (func_avg.go:53)
    assert agg(data[2:], tp, [(SUM, 0), (AVG, 0)])[1] == [(conv(9), conv(3))]
    rc, rows = agg(data + data[2:], tp, [(SUM, 0), (AVG, 0), (COUNT, 0)])
    assert rows == [(conv(19), 2 if tp == INT64 else 2.375, 8)]
    # NULL rows are skipped; an all-NULL input stays NULL (aggfunc_test.go:184-190 appends a NULL row)
    assert agg(data + [None], tp, [(SUM, 0), (COUNT, 0), (COUNT, -1)])[1] == [(conv(10), 5, 6)]
    assert agg([None, None], tp, [(SUM, 0), (AVG, 0), (MAX, 0), (COUNT, 0)])[1] == [(N, N, N, 0)]


def test_max_min_first_row_goldens():
    # func_max_min_test.go: 0..4 -> max 4 / min 0; merge with rows 2..4 -> max 4 / min 0;  first_row -> 0 then 2
    data = list(range(5))
    assert agg(data, INT64, [(MAX, 0), (MIN, 0), (FIRSTROW, 0)])[1] == [(4, 0, 0)]
    assert agg(data[2:], INT64, [(MAX, 0), (MIN, 0), (FIRSTROW, 0)])[1] == [(4, 2, 2)]
    assert agg([1.5, -2.5, None], FLOAT64, [(MAX, 0), (MIN, 0)])[1] == [(1.5, -2.5)]
    u = [1, (1 << 64) - 1, 5]
    cols = [Column(UINT64, np.array(u, dtype=np.uint64))]
    assert O.hash_agg([UINT64], cols, [], [(MAX, 0), (MIN, 0)])[1].rows() == [((1 << 64) - 1, 1)]
    # executor/aggregate_test.go:74-81 TestAggEliminator: min/max over (1,-1),(2,-2),(3,1),(4,NULL); b*b pre-projected
    b = [-1, -2, 1, None]
    assert agg(b, INT64, [(MIN, 0)])[1] == [(-2,)]
    assert agg([1, 4, 1, None], INT64, [(MAX, 0), (MIN, 0)])[1] == [(4, 1)]
    assert agg([], INT64, [(MIN, 0), (MIN, 0)])[1] == [(N, N)]


def test_group_by_goldens():
    # executor/aggregate_test.go:51-69 TestAggPushDown
    assert agg([], INT64, [(COUNT, 0)], group=[]) == (0, [])                   # count(a) from t group by a (empty) -> no rows
    assert agg([], INT64, [(COUNT, 0)]) == (0, [(0,)])                         # count(a) from t (empty) -> 0
    assert agg([0], INT64, [(COUNT, 0)], group=[0]) == (0, [(1,)])             # one row
    # rows (a,b): (0,0),(1,1),(3,3),(3,2),(2,1),(1,1),(1,1); where b>0; count(a) group by a,b -> sorted 1,1,1,3
    rows = [(1, 1), (3, 3), (3, 2), (2, 1), (1, 1), (1, 1)]
    a = [r[0] for r in rows]
    ab = [r[0] * 100 + r[1] for r in rows]  # the pair (a,b) folded into one key column (single GROUP BY column in this round)
    rc, out = agg(a, INT64, [(COUNT, 0)], group=ab)
    assert sorted(r[0] for r in out) == [1, 1, 1, 3]
    # executor/executor_test.go:964-977: count(*), c group by c / sum(c) group by b — NULL is its own group
    rc, out = agg([1, 1, None, None, 2], INT64, [(COUNT, -1), (FIRSTROW, 0)], group=[1, 1, 7, 7, 2])
    assert sorted(out, key=str) == sorted([(2, 1), (2, None), (1, 2)], key=str)
    rc, out = O.hash_agg([INT64], [icol([1, N, 1, N])], [0], [(COUNT, -1), (FIRSTROW, 0)], 1)
    assert sorted(out.rows(), key=str) == sorted([(2, 1), (2, None)], key=str)


def test_int_sum_overflow_is_an_error():
    # types.AddInt64 (types/overflow.go:33-40) via func_sum.go:133
    big = (1 << 63) - 1
    assert agg([big, 1], INT64, [(SUM, 0)])[0] == 3
    assert agg([-big - 1, -1], INT64, [(AVG, 0)])[0] == 3
    assert agg([big, -1], INT64, [(SUM, 0)]) == (0, [(big - 1,)])


@pytest.mark.parametrize("workers", [1, 2, 4, 7])
def test_partial_final_split_is_result_neutral(workers):
    # AggFuncDesc.Split (expression/aggregation/descriptor.go:57-92): any number of partial workers, same answer
    rng = np.random.default_rng(11)
    n = 20000
    k = Column(INT64, rng.integers(0, 300, n), rng.random(n) > 0.05)
    v = Column(INT64, rng.integers(-1000, 1000, n), rng.random(n) > 0.1)
    f = Column(FLOAT64, np.floor(rng.random(n) * 1024) / 8, rng.random(n) > 0.1)  # dyadic: float sums are exact in any order
    funcs = [(COUNT, -1), (COUNT, 1), (SUM, 1), (AVG, 1), (MAX, 1), (MIN, 1), (SUM, 2), (AVG, 2), (MAX, 2), (FIRSTROW, 0)]
    rc1, base = O.hash_agg([INT64, INT64, FLOAT64], [k, v, f], [0], funcs, 1)
    rc2, other = O.hash_agg([INT64, INT64, FLOAT64], [k, v, f], [0], funcs, workers)
    assert rc1 == rc2 == 0
    key = lambda r: (r[-1] is None, r[-1] or 0)
    assert sorted(base.rows(), key=key) == sorted(other.rows(), key=key)


# ------------------------------------------------------------------ the multi-threaded CPU baseline agrees with the oracle
def test_cpu_reference_design_matches_oracle():
    rng = np.random.default_rng(5)
    nb, npr = 50000, 200000
    bk = rng.permutation(nb).astype(np.int64)
    bk[:100] = bk[100:200]  # some duplicate build keys
    bv = bk * 7 + 1
    pk = rng.integers(0, nb + 1000, npr).astype(np.int64)
    pv = np.arange(npr, dtype=np.int64)
    lib = O.load()
    bs, ps, ck = C.c_double(0), C.c_double(0), C.c_uint64(0)
    rows = lib.orc_mt_join_bench(C.c_int64(nb), C.c_void_p(bk.ctypes.data), C.c_void_p(bv.ctypes.data), C.c_int64(npr), C.c_void_p(pk.ctypes.data),
                                 C.c_void_p(pv.ctypes.data), C.c_int(4), C.byref(bs), C.byref(ps), C.byref(ck))
    want = O.hash_join(INNER, True, [INT64, INT64], [Column(INT64, bk), Column(INT64, bv)], [INT64, INT64], [Column(INT64, pk), Column(INT64, pv)], [0], [0])
    assert rows == want.num_rows()
    exp = int(np.sum((want.cols[1].values.view(np.uint64) ^ want.cols[3].values.view(np.uint64)).astype(np.uint64), dtype=np.uint64))
    assert ck.value == exp
    # group-by baseline
    n = 300000
    k = rng.integers(0, 5000, n).astype(np.int64)
    x = (np.floor(rng.random(n) * 1024) / 8).astype(np.float64)
    sec, ss, sc = C.c_double(0), C.c_double(0), C.c_int64(0)
    groups = lib.orc_mt_agg_bench(C.c_int64(n), C.c_void_p(k.ctypes.data), C.c_void_p(x.ctypes.data), C.c_int(4), C.c_int(4), C.byref(sec), C.byref(ss), C.byref(sc))
    assert groups == len(np.unique(k)) and sc.value == n and ss.value == float(x.sum())
