"""GPU suite: the GROUP BY across ranks (tq_agg_push_partial[_var] -> tq_region_wait -> tq_agg_merge_regions[_var]) at the
int64 limits and at the order-free DOUBLE bound, with W ranks emulated in one process on exchange_ref's sentinel-guarded
Regions.

A partial row carries a 64-bit total while the single-GPU state is 128 bits, so the range rule (DESIGN §3 deviation i) splits:
a part of one group on one rank that leaves int64 fails that rank's push, and then every destination's merge; a merged total
that leaves int64 fails only the rank that finishes the group.  The families of tests/int_agg_ref.py are dealt over the ranks
(int_agg_ref.deal) and every rank's result is compared bit for bit with region_agg_ref.expect_ranks, which names where each
failure lands.  DOUBLE SUM / AVG are held to float_agg_ref.check_sum.  FLOAT (float32) is not covered: device puts refuse
it, and the region path takes device columns only."""
import numpy as np
import pytest

import exchange_ref as X
import float_agg_ref as F
import int_agg_ref as I
import region_agg_ref as RA
import region_agg_strings_ref as S
import region_outer_ref as R
from test_gpu_float_agg import check as float_check
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, FLOAT64, INT64, UINT64, Chunk, Column, VarColumn
from tinysql_b200.dist import RegionAgg, partial_var_cols

pytestmark = pytest.mark.gpu

COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)
WS = [1, 2, 3, 8]
FUNCS = [(COUNT, -1), (COUNT, 1), (SUM, 1), (AVG, 1), (MAX, 1), (MIN, 1), (FIRSTROW, 1), (FIRSTROW, 0)]
OVF = L.TQ_ERR_OVERFLOW_BIGINT
FAILED = 0xFFFFFFFF00000000


@pytest.fixture(scope="module")
def lib():
    lib = L.load()
    L.check(lib.tq_init(0))
    return lib


def _int_cols(d, tp):
    return [I.key_column(d.gid) if len(d.gid) else Column(INT64, np.zeros(0, np.int64), np.zeros(0, bool)), Column(tp, d.x, d.nn)]


def _str_cols(d, tp):
    """the same groups keyed by a VARCHAR: group id g -> b"g<g>" ("" for 0, NULL for 5)"""
    keys = [None if g == 5 else (b"" if g == 0 else b"g%d" % g) for g in d.gid.tolist()]
    return [VarColumn(BYTES, keys), Column(tp, d.x, d.nn)]


def _step(lib, W, types, group_by, funcs, rank_cols, reg=None, epoch=1, var=False):
    """one step over emulated ranks (on reg, or on fresh regions sized for rank_cols); returns (push statuses, per
    destination (merge status, next status, Columns or None)) as region_agg_ref.run(statuses=True)"""
    own = reg is None
    if reg is None:
        reg = _regions(lib, W, types, group_by, funcs, rank_cols, var)
    if var:
        shards = [S.device(cols) for cols in rank_cols]
    else:
        shards = [R.Source(lib, [np.ascontiguousarray(c.values).view(np.uint64) for c in cols], [c.not_null() for c in cols]) for cols in rank_cols]
    try:
        return RA.run(lib, W, types, group_by, funcs, shards, reg, epoch, statuses=True, byte_cap=reg.byte_cap if var else None)
    finally:
        for sh in shards:
            for c in (sh if var else [sh]):
                c.free()
        if own:
            reg.free()


def _regions(lib, W, types, group_by, funcs, rank_cols, var=False):
    w = RA.width(lib, RA.desc(types, group_by, funcs)[0])
    groups = max(c[0].length for c in rank_cols) + 1
    if not var:
        return X.Regions(lib, W, w + 1, groups + 8)
    caps = S.byte_caps(types, group_by, funcs, rank_cols)
    (nc, cap, words), byte_cap = RegionAgg.table_of(W, w, partial_var_cols(types, group_by, funcs), bool(group_by), groups, caps)
    reg = X.Regions(lib, W, nc, cap, words=words)
    reg.byte_cap = byte_cap
    return reg


def _key_idx(funcs, group_by):
    return [i for i, (f, a) in enumerate(funcs) if f == FIRSTROW and a in group_by]


def _assert_ranks(exp, pushed, out, funcs, group_by, W):
    """statuses where expect_ranks puts them, and every other rank's groups exact (and only its own)"""
    want_push = [OVF if s in exp.push_fail else L.TQ_OK for s in range(W)]
    assert pushed == want_push, (pushed, want_push)
    for q, (merge, nxt, cols) in enumerate(out):
        if exp.push_fail:
            assert merge == OVF and cols is None, (q, merge)
            continue
        assert merge == L.TQ_OK, (q, merge)
        if q in exp.dest_fail:
            assert nxt == OVF, (q, nxt)
            continue
        assert nxt == L.TQ_OK, (q, nxt)
        if not group_by and q:
            assert cols is None, "a scalar aggregate is finished on rank 0 only"
            continue
        got = I.result_rows(Chunk(cols), _key_idx(funcs, group_by))
        bad = I.mismatches(got, exp.ranks[q], funcs)
        assert not bad, (q, len(bad), bad[:5])


def _run_dealt(lib, W, dealt, tp, group_by=(0,), funcs=FUNCS, var=False):
    cols_of = _str_cols if var else _int_cols
    rank_cols = [cols_of(d, tp) for d in dealt]
    types = [BYTES if var else INT64, tp]
    exp = RA.expect_ranks(types, rank_cols, list(group_by), funcs, W)
    pushed, out = _step(lib, W, types, list(group_by), funcs, rank_cols, var=var)
    _assert_ranks(exp, pushed, out, funcs, list(group_by), W)
    return exp


def _with_lonely_argument(dealt, W, empty, tp):
    """one more group with rows on every rank that holds rows, its argument NULL on all of them but one"""
    g = max(int(d.gid.max()) for d in dealt if len(d.gid)) + 1
    out, first = [], True
    for r, d in enumerate(dealt):
        if r in empty:
            out.append(d)
            continue
        nn = np.array([first] * 3)
        first = False
        out.append(I.Dealt(np.append(d.gid, [g] * 3), np.append(d.x, np.array([7, 7, 7], dtype=d.x.dtype)), np.append(d.nn, nn), d.parts))
    return out


INT_FAMILIES = ["limits", "prefix_wraps", "unsigned", "avg_trunc", "extremes_only_int64", "extremes_only_uint64"]


def _family(name, rng):
    if name.startswith("extremes_only"):
        return I.check_family(I.extremes_only(rng, UINT64 if name.endswith("uint64") else INT64))
    return I.check_family(I.make(name, rng))


@pytest.mark.parametrize("W", WS)
@pytest.mark.parametrize("name", INT_FAMILIES)
def test_int_families_dealt_over_ranks(lib, name, W):
    """every family exact on every rank, each group finished once on the rank its key names: COUNT(*), COUNT, SUM, AVG, MAX,
    MIN, FIRSTROW(x) (a value of its group), FIRSTROW(key) over the edge keys and NULL; rank 1 holds nothing when W >= 3"""
    rng = np.random.default_rng(10 * INT_FAMILIES.index(name) + W)
    fam = _family(name, rng)
    tp = UINT64 if fam.x.dtype == np.uint64 else INT64
    empty = (1,) if W >= 3 else ()
    dealt = I.deal(rng, fam, W, rebuild=name == "limits", whole=name == "prefix_wraps", empty=empty)
    dealt = _with_lonely_argument(dealt, W, empty, tp)
    exp = _run_dealt(lib, W, dealt, tp)
    assert not exp.push_fail and not exp.dest_fail


@pytest.mark.parametrize("func", [SUM, AVG])
@pytest.mark.parametrize("twin,W", [(t, W) for t in sorted(I.TWINS) for W in (2, 3, 8) if W > 2 or "2_64" not in t])
def test_merged_total_past_the_limit_fails_its_rank_only(lib, twin, W, func):
    """every part in range, one group's merged total one past a limit (or ±2^64, which needs 3 in-range parts): exactly the
    rank that finishes it fails with TQ_ERR_OVERFLOW_BIGINT from next, the others are exact; the in-range twin is exact
    everywhere"""
    rng = np.random.default_rng(300 + W + 10 * func)
    fam = I.limits(rng, n_groups=120, hi=600)
    funcs = [(COUNT, -1), (func, 1), (FIRSTROW, 0)]
    exp = _run_dealt(lib, W, I.deal(rng, fam, W, rebuild=True), INT64, funcs=funcs)
    assert not exp.push_fail and not exp.dest_fail
    bad = I.check_family(I.out_by_one(fam, I.TWINS[twin], rng))
    dealt = I.deal(rng, bad, W, rebuild=True)
    assert all(I.in_range(t) for d in dealt for t in d.parts.values())
    exp = _run_dealt(lib, W, dealt, INT64, funcs=funcs)
    assert not exp.push_fail and len(exp.dest_fail) == 1


def _big_group(fam):
    sizes, tot = np.bincount(fam.gid), I.group_totals(fam)
    return max((g for g in range(len(sizes)) if tot[g] >= 0), key=lambda g: sizes[g])


@pytest.mark.parametrize("key", ["int64", "varchar"])
def test_part_past_the_limit_fails_every_rank_then_the_next_step_runs(lib, key):
    """one source's part of one group totals INT64_MAX + 1 while the merged total is in range: that push returns
    TQ_ERR_OVERFLOW_BIGINT, writes no region row and marks its slot on every rank under the step's epoch; every merge
    refuses the step; the other sources' slots and rows are what they would have been; a clean step at the next epoch on
    the same regions is exact"""
    W, src = 3, 1
    var = key == "varchar"
    rng = np.random.default_rng(500 + var)
    fam = I.limits(rng, n_groups=150, hi=500)
    g = _big_group(fam)
    seed = int(rng.integers(1 << 30))
    bad = I.deal(np.random.default_rng(seed), fam, W, rebuild=True, past=(g, src))
    good = I.deal(np.random.default_rng(seed), fam, W, rebuild=True)
    funcs = [(COUNT, -1), (SUM, 1), (FIRSTROW, 0)]
    cols_of = _str_cols if var else _int_cols
    types = [BYTES if var else INT64, INT64]
    bad_cols, good_cols = [cols_of(d, INT64) for d in bad], [cols_of(d, INT64) for d in good]
    exp = RA.expect_ranks(types, bad_cols, [0], funcs, W)
    assert exp.push_fail == {src}
    reg = _regions(lib, W, types, [0], funcs, bad_cols + good_cols, var)
    try:
        pushed, out = _step(lib, W, types, [0], funcs, bad_cols, reg=reg, epoch=1, var=var)
        _assert_ranks(exp, pushed, out, funcs, [0], W)
        for q in range(W):
            slots = reg.slots(q)
            assert slots[src] == (FAILED | OVF, 1), (q, slots[src])
            for c in range(reg.ncols[0]):
                assert np.all(reg.region(q, src, c) == X.SENTINEL), f"the failed source wrote region {q}, column {c}"
            for s in range(W):
                if s == src:
                    continue
                want = _wire_rows(bad_cols[s], types, funcs, W, q)
                assert slots[s] == (len(want), 1), (q, s, slots[s], len(want))
                if not var:
                    got = np.stack([reg.region(q, s, c)[:len(want)] for c in range(reg.ncols[0])], 1)
                    assert np.array_equal(X.sorted_rows(_canon_wire(got)), X.sorted_rows(want)), (q, s)
        exp = RA.expect_ranks(types, good_cols, [0], funcs, W)
        pushed, out = _step(lib, W, types, [0], funcs, good_cols, reg=reg, epoch=2, var=var)
        _assert_ranks(exp, pushed, out, funcs, [0], W)
        assert all(st == L.TQ_OK for st in pushed) and all(m == L.TQ_OK and n == L.TQ_OK for m, n, _ in out)
    finally:
        reg.free()


def _canon_wire(m):
    """wire rows with the words of NULL cells zeroed (their bits are not promised)"""
    m = m.copy()
    mask = m[:, -1]
    for c in range(m.shape[1] - 1):
        m[:, c] = np.where((mask >> np.uint64(c)) & np.uint64(1), m[:, c], np.uint64(0))
    return m


def _wire_rows(cols, types, funcs, W, q):
    """the partial rows of one source that go to destination q, as wire words (key, states in function order, mask; NULL
    cells 0), from int_agg_ref.expect_partial (states first, then the key)"""
    if not cols[0].length:
        return np.zeros((0, 5), np.uint64)
    _, ch = I.expect_partial(types, cols, [0], funcs)
    vals = [c.tolist() for c in ch.cols]
    keys = vals[-1]
    d = RA.key_dest([(k,) for k in keys], [types[0]], W)
    rows = []
    for i in np.nonzero(d == q)[0]:
        cells = [keys[i]] + [v[i] for v in vals[:-1]]
        mask = sum(1 << c for c, v in enumerate(cells) if v is not None)
        rows.append([v % (1 << 64) if isinstance(v, int) else 0 for v in cells] + [mask])   # a string key: counted only
    return np.array(rows, dtype=object).astype(np.uint64).reshape(-1, 5)


@pytest.mark.parametrize("W", [1, 3, 8])
@pytest.mark.parametrize("total", [I.INT64_MAX, I.INT64_MIN, I.INT64_MAX + 1])
def test_scalar_aggregate_at_the_limits(lib, W, total):
    """no GROUP BY: the ranks' parts total exactly INT64_MAX, INT64_MIN or one past; only rank 0 finishes, and only rank 0
    fails (with one rank the one part is past the limit, so its push fails)"""
    rng = np.random.default_rng(700 + W)
    m = 40 * W
    fam = I.Family("scalar", np.zeros(m, np.int64), np.array(I.group_terms(rng, m, total), dtype=object).astype(np.int64),
                   np.ones(m, bool), {})
    dealt = I.deal(rng, fam, W, rebuild=True)
    rank_cols = [[Column(INT64, d.x, d.nn)] for d in dealt]
    funcs = [(COUNT, -1), (SUM, 0), (AVG, 0), (MAX, 0), (MIN, 0)]
    exp = RA.expect_ranks([INT64], rank_cols, [], funcs, W)
    pushed, out = _step(lib, W, [INT64], [], funcs, rank_cols)
    _assert_ranks(exp, pushed, out, funcs, [], W)
    past = not I.in_range(total)
    assert exp.dest_fail == ({0} if past and W > 1 else set()) and exp.push_fail == ({0} if past and W == 1 else set())


@pytest.mark.parametrize("W", WS)
@pytest.mark.parametrize("family", ["tight", "ill", "subnormal", "overflow", "zeros"])
def test_double_families_dealt_over_ranks(lib, family, W):
    """DOUBLE SUM / AVG within the order-free bound (subnormal bit-equal, overflow exactly ±inf, a group of zeros +0.0),
    COUNT / MAX / MIN as the oracle with -0.0 < +0.0, each group once on its rank"""
    rng = np.random.default_rng(900 + W)
    n = 40_000
    gid = rng.integers(0, 700, n)
    if family == "overflow":
        gid = rng.integers(0, 4000, n)   # groups of a few rows: both sides of the 3 / 4 row line
    x = F.family_column(family, rng, gid)
    keys = I.key_column(gid)
    rank = rng.integers(0, W, n)
    rank_cols = []
    for r in range(W):
        sel = np.nonzero(rank == r)[0]
        rank_cols += [[Column(INT64, keys.values[sel], keys.not_null()[sel]), Column(FLOAT64, x.values[sel], x.not_null()[sel])]]
    types = [INT64, FLOAT64]
    funcs = [(COUNT, -1), (COUNT, 1), (SUM, 1), (AVG, 1), (MAX, 1), (MIN, 1), (FIRSTROW, 0)]
    pushed, out = _step(lib, W, types, [0], funcs, rank_cols)
    assert all(st == L.TQ_OK for st in pushed) and all(m == L.TQ_OK and nx == L.TQ_OK for m, nx, _ in out)
    for q, (_, _, cols) in enumerate(out):
        if cols[0].length:
            assert np.all(RA.key_dest([(k,) for k in cols[6].tolist()], [INT64], W) == q), f"rank {q} finished another rank's group"
    got = Chunk.concat([Chunk(c) for _, _, c in out], [c.tp for c in out[0][2]])
    order = np.argsort(rank, kind="stable")
    all_cols = [Column(INT64, keys.values[order], keys.not_null()[order]), Column(FLOAT64, x.values[order], x.not_null()[order])]
    exact = float_check(got, types, all_cols, [0], funcs, family)
    if family == "tight":   # a dropped, doubled or misrouted row must fail check_sum
        F.assert_sensitive(exact)


def test_string_key_at_the_limits(lib):
    """GROUP BY a VARCHAR with SUM / AVG of the limits family through tq_agg_push_partial_var / tq_agg_merge_regions_var"""
    W = 3
    rng = np.random.default_rng(1100)
    fam = I.check_family(I.limits(rng, n_groups=200, hi=800))
    dealt = I.deal(rng, fam, W, rebuild=True)
    funcs = [(COUNT, -1), (SUM, 1), (AVG, 1), (MAX, 1), (FIRSTROW, 0)]
    exp = _run_dealt(lib, W, dealt, INT64, funcs=funcs, var=True)
    assert not exp.push_fail and not exp.dest_fail
