"""CPU suite: the exact BIGINT / BIGINT UNSIGNED aggregation reference of tests/int_agg_ref.py and its aimed datasets.

The reference must equal the oracle wherever the two contracts agree (every in-order prefix of every group in range), must
reproduce the reference's own TestSum / TestAvg / TestAvgFinalMode answers, and every dataset family must reach the edge it
is named after; prefix_wraps must make the oracle raise, which is what keeps it aimed at DESIGN §3 deviation (i)."""
import numpy as np
import pytest

import int_agg_ref as R
import oracle_py as O
from tinysql_b200.chunk import INT64, UINT64, Column

COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)
FUNCS = [(COUNT, -1), (COUNT, 1), (SUM, 1), (AVG, 1), (MAX, 1), (MIN, 1), (FIRSTROW, 1), (FIRSTROW, 0)]


def _all_prefixes_in_range(gid, x, nn):
    order = np.argsort(gid[nn], kind="stable")
    g, v = gid[nn][order], np.asarray(x)[nn][order]
    starts = np.searchsorted(g, np.unique(g))
    return not any(R.prefix_out_of_range(seg).any() for seg in np.split(v, starts[1:]))


def _cases():
    rng = np.random.default_rng(5)
    n = 30_000
    gid = rng.integers(0, 400, n)
    yield "small", gid, Column(INT64, rng.integers(-(1 << 40), 1 << 40, n), rng.random(n) >= 0.1)
    u = np.where(rng.random(n) < 0.5, rng.integers(0, 1 << 40, n).astype(np.uint64),
                 np.uint64(R.UINT64_MAX) - rng.integers(0, 1 << 40, n).astype(np.uint64))
    yield "unsigned_small", gid, Column(UINT64, u, rng.random(n) >= 0.1)   # both sides of 2^63, small int64 readings
    for tp in (INT64, UINT64):
        f = R.check_family(R.extremes_only(rng, tp))
        yield f"extremes_{tp}", f.gid, Column(tp, f.x, f.nn)


@pytest.mark.parametrize("case", ["small", "unsigned_small", f"extremes_{INT64}", f"extremes_{UINT64}"])
@pytest.mark.parametrize("workers", [1, 3])
def test_reference_equals_oracle_where_prefixes_are_in_range(case, workers):
    name, gid, x = next(c for c in _cases() if c[0] == case)
    assert _all_prefixes_in_range(gid, x.values, x.not_null())
    k = R.key_column(gid)
    types, cols = [INT64, x.tp], [k, x]
    want = R.expect(cols, [0], FUNCS)
    assert not want.overflow
    rc, got = O.hash_agg(types, cols, [0], FUNCS, workers)
    assert rc == 0
    assert R.mismatches(R.result_rows(got, [7]), want, FUNCS) == []
    # no GROUP BY: one group (the extremes of both signs leave int64 on the way there)
    one = np.zeros_like(gid)
    assert _all_prefixes_in_range(one, x.values, x.not_null()) == case.startswith(("small", "unsigned"))
    if not case.startswith(("small", "unsigned")):
        return
    want = R.expect(cols, [], FUNCS[:6])
    rc, got = O.hash_agg(types, cols, [], FUNCS[:6], workers)
    assert rc == 0 and R.mismatches(R.result_rows(got, []), want, FUNCS[:6]) == []


def _one(vals, funcs, tp=INT64):
    x = R.column(tp, vals)
    want = R.expect([x], [], funcs)
    return want.overflow, want.groups[()]


def test_reference_reproduces_the_sum_avg_goldens():
    data = list(range(5))
    # func_sum_test.go TestSum / func_avg_test.go TestAvg (as test_oracle_golden.py transcribes them)
    assert _one([], [(SUM, 0), (AVG, 0), (COUNT, 0)]) == (False, [None, None, 0])
    assert _one(data, [(SUM, 0), (AVG, 0), (COUNT, 0)]) == (False, [10, 2, 5])
    assert _one(data[2:], [(SUM, 0), (AVG, 0)]) == (False, [9, 3])
    assert _one(data + data[2:], [(SUM, 0), (AVG, 0), (COUNT, 0)]) == (False, [19, 2, 8])   # 19 / 8 truncates to 2
    assert _one(data + [None], [(SUM, 0), (COUNT, 0), (COUNT, -1)]) == (False, [10, 5, 6])
    assert _one([None, None], [(SUM, 0), (AVG, 0), (MAX, 0), (COUNT, 0)]) == (False, [None, None, None, 0])
    # types.AddInt64 overflow, and a total back in range
    big = R.INT64_MAX
    assert _one([big, 1], [(SUM, 0)])[0] and _one([-big - 1, -1], [(AVG, 0)])[0]
    assert _one([big, -1], [(SUM, 0)]) == (False, [big - 1])
    # Go's integer division truncates toward zero
    assert _one([-7, 0], [(AVG, 0)]) == (False, [-3]) and _one([-7, 0, 0], [(AVG, 0)]) == (False, [-2])
    assert _one([R.INT64_MIN, 0, 0], [(AVG, 0)]) == (False, [-3074457345618258602])
    # MAX / MIN: unsigned order for BIGINT UNSIGNED (func_max_min_test.go), and an unsigned SUM argument read as int64
    assert _one([1, R.UINT64_MAX, 5], [(MAX, 0), (MIN, 0), (SUM, 0)], UINT64) == (False, [R.UINT64_MAX, 1, 5])
    assert _one([1 << 63, (1 << 63) - 1], [(MAX, 0), (MIN, 0), (SUM, 0)], UINT64) == (False, [1 << 63, (1 << 63) - 1, -1])


def test_reference_reproduces_the_avg_final_mode_golden():
    # TestAvgFinalMode: partial rows (count i, sum i*i), i = 1..100 -> 338350 / 5050 = 67
    i = np.arange(1, 101, dtype=np.int64)
    want = R.expect_final([Column(INT64, i), Column(INT64, i * i)], [], [(AVG, 0, 1)])
    assert want == R.Expected({(): [67]}, False)
    # a partial row with a NULL sum is skipped together with its count (func_avg.go:96-110)
    cnt, s = Column(INT64, [2, 5, 0]), Column(INT64, [3, 0, 0], [True, False, False])
    want = R.expect_final([cnt, s], [], [(AVG, 0, 1), (COUNT, 0, -1), (SUM, 1, -1)])
    assert want == R.Expected({(): [1, 7, 3]}, False)
    rc, got = O.hash_agg_final([INT64, INT64], [cnt, s], [], [(AVG, 0, 1), (COUNT, 0, -1), (SUM, 1, -1)])
    assert rc == 0 and got.rows() == [(1, 7, 3)]


def test_final_of_reference_partials_equals_complete():
    """Final(Partial1(region 1) ++ Partial1(region 2) ++ Partial1(region 3)) == Complete(all rows), and it agrees with the
    oracle's FinalMode, on data whose regions' totals stay in range"""
    rng = np.random.default_rng(9)
    n = 20_000
    gid = rng.integers(0, 300, n)
    k = R.key_column(gid)
    for x in (Column(INT64, rng.integers(-(1 << 58), 1 << 58, n), rng.random(n) >= 0.2),
              Column(UINT64, np.where(rng.random(n) < 0.5, np.uint64(0), np.uint64(R.UINT64_MAX - (1 << 56))) + rng.integers(0, 1 << 56, n).astype(np.uint64),
                     rng.random(n) >= 0.2)):
        funcs = [(COUNT, 1), (SUM, 1), (AVG, 1), (MAX, 1), (MIN, 1), (FIRSTROW, 0)]
        types = [INT64, x.tp]
        whole = R.expect([k, x], [0], funcs)
        regions = [0, 4000, 4100, n]
        parts = [R.expect_partial(types, [c.slice(lo, hi) for c in (k, x)], [0], funcs) for lo, hi in zip(regions[:-1], regions[1:])]
        ptypes = parts[0][0]
        pcols = [Column(t, np.concatenate([p[1].cols[c].values for p in parts]), np.concatenate([p[1].cols[c].not_null() for p in parts]))
                 for c, t in enumerate(ptypes)]
        ff, pgb = R.final_funcs(funcs, 1)
        assert (ff, pgb) == ([(COUNT, 0, -1), (SUM, 1, -1), (AVG, 2, 3), (MAX, 4, -1), (MIN, 5, -1), (FIRSTROW, 6, -1)], [7])
        got = R.expect_final(pcols, pgb, ff)
        assert got.overflow == whole.overflow
        assert set(got.groups) == set(whole.groups)
        for key, w in whole.groups.items():
            assert got.groups[key][:5] == w[:5], key
            assert got.groups[key][5] == frozenset([key[0]])
        if not whole.overflow:
            rc, orc = O.hash_agg_final(ptypes, pcols, [7], ff)
            assert rc == 0 and R.mismatches(R.result_rows(orc, [5]), got, ff) == []


@pytest.mark.parametrize("name", R.FAMILIES)
def test_family_self_check(name):
    R.check_family(R.make(name, np.random.default_rng(R.FAMILIES.index(name))))


def test_extremes_unsigned_self_check():
    R.check_family(R.extremes_only(np.random.default_rng(3), UINT64))


@pytest.mark.parametrize("twin", sorted(R.TWINS))
def test_out_by_one_twin_self_check(twin):
    rng = np.random.default_rng(17)
    base = R.check_family(R.limits(rng, 90, 2, 400))
    t = R.check_family(R.out_by_one(base, R.TWINS[twin], rng))
    g = t.meta["group"]
    assert (t.x != base.x).sum() >= 1 and np.array_equal(t.x[t.gid != g], base.x[base.gid != g])
    cols = [R.key_column(t.gid), Column(INT64, t.x)]
    funcs = [(SUM, 1), (AVG, 1), (FIRSTROW, 0)]
    assert R.expect(cols, [0], funcs).overflow
    assert not R.expect([R.key_column(base.gid), Column(INT64, base.x)], [0], funcs).overflow
    if twin in ("plus_2_64", "minus_2_64"):
        assert R.group_totals(t)[g] % (1 << 64) == 0   # the low word of the exact total is 0


def test_prefix_wraps_makes_the_oracle_raise():
    f = R.check_family(R.prefix_wraps(np.random.default_rng(4), 60))
    cols = [R.key_column(f.gid), Column(INT64, f.x)]
    assert not R.expect(cols, [0], [(SUM, 1)]).overflow
    assert O.hash_agg([INT64, INT64], cols, [0], [(SUM, 1)])[0] == 3
    for g in range(0, 60, 7):   # and group by group, with one partial worker each
        x = Column(INT64, f.x[f.gid == g])
        assert O.hash_agg([INT64], [x], [], [(AVG, 0)])[0] == 3, g


def test_key_column_keeps_the_edge_keys_apart():
    gid = np.arange(40)
    k = R.key_column(gid)
    vals = k.tolist()
    assert vals[:6] == R.EDGE_KEYS + [None]
    assert len(set(vals)) == 40
