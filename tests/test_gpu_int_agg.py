"""BIGINT / BIGINT UNSIGNED COUNT, SUM, AVG, MAX, MIN and FIRSTROW on every aggregation path against the exact reference of
tests/int_agg_ref.py, at the int64 limits.

Each dataset family (limits, prefix_wraps, unsigned, avg_trunc, extremes_only; GROUP BY keys INT64_MIN, INT64_MAX, -1, 0,
NULL and the table's free-slot marker among them) runs through the general update with divergent and warp-uniform warps,
the 8e6-row scalar aggregate, the NOT NULL compact state and the flag back-fill, table growth with deferred replay,
multi-column and VARCHAR GROUP BYs, device input, export / merge, FinalMode and the pre-aggregation decision.  Values are
compared bit for bit and NULL masks exactly; FIRSTROW of a non-key column may be any row of its group (deviation ii).

The range check is pinned from both sides: every out_by_one twin (one group's exact total at INT64_MAX + 1, INT64_MIN - 1 or
±2^64, every other row unchanged) must fail with ErrOverflow, and its in-range twin must give exact values.  The
prefix_wraps family makes the C oracle raise (it adds in row order); the device must not (DESIGN §3 deviation i)."""
import ctypes as C

import numpy as np
import pytest

import int_agg_ref as R
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, INT64, UINT64, Column, DeviceColumn, tq_array
from tinysql_b200.executor import HashAggExec, HashAggFinalExec, MockDataSource

pytestmark = pytest.mark.gpu

COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)
SWITCHES = ("TQ_AGG_NO_PREAGG", "TQ_AGG_PREAGG_PART")
FAMS = R.FAMILIES


def _switches(monkeypatch, env):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _stats(lib, e):
    st = (C.c_int64 * 4)()
    L.check(lib.tq_agg_stats(e.handle, st))
    return list(st)


def _empty(types):
    return MockDataSource(types, [Column(t, [] if t == BYTES else np.zeros(0)) for t in types])


def run_host(lib, types, cols, gb, funcs, est, not_null=(), chunk=1 << 16):
    e = HashAggExec(MockDataSource(types, cols, chunk), gb, funcs, est, not_null_cols=not_null)
    e.Open()
    try:
        got = e.drain()
        return got, _stats(lib, e)
    finally:
        e.Close()


def run_device(lib, types, batches, gb, funcs, est, not_null=(), launches=None):
    """one TQ_MEM_DEVICE put per batch (a column without a bitmap goes in without one); `launches` collects the handle's
    launch count after each put"""
    e = HashAggExec(_empty(types), gb, funcs, est, not_null_cols=not_null)
    e.Open()
    try:
        for cols in batches:
            d = [DeviceColumn.from_host(c) for c in cols]
            try:
                L.check(lib.tq_agg_put(e.handle, (L.TQColumn * len(d))(*[x.tq() for x in d]), L.TQ_MEM_DEVICE))
            finally:
                for x in d:
                    x.free()
            if launches is not None:
                launches.append(_stats(lib, e)[3])
        got = e.drain()
        return got, _stats(lib, e)
    finally:
        e.Close()


def run_export_merge(lib, types, parts, gb, funcs, est):
    """one Partial1 handle per part -> tq_agg_export_partial -> tq_agg_merge_partial into one handle"""
    final = HashAggExec(_empty(types), gb, funcs, est)
    final.Open()
    try:
        width = C.c_int32(0)
        L.check(lib.tq_agg_partial_width(final.handle, C.byref(width)))
        for cols in parts:
            part = HashAggExec(MockDataSource(types, cols, 1 << 16), gb, funcs, est)
            part.Open()
            try:
                while True:
                    chk = part.child.Next()
                    if chk.num_rows() == 0:
                        break
                    L.check(lib.tq_agg_put(part.handle, tq_array(chk.cols), L.TQ_MEM_HOST))
                out = (L.TQColumn * width.value)()
                rows = C.c_int64(0)
                L.check(lib.tq_agg_export_partial(part.handle, out, C.byref(rows)))
                L.check(lib.tq_agg_merge_partial(final.handle, out, L.TQ_MEM_DEVICE))
            finally:
                part.Close()
        return final.drain()
    finally:
        final.Close()


def run_final(ptypes, pcols, pgb, ffuncs):
    e = HashAggFinalExec(MockDataSource(ptypes, pcols, 1000), pgb, ffuncs, 0)
    e.Open()
    try:
        return e.drain()
    finally:
        e.Close()


def raises_overflow(fn, *args, **kw):
    with pytest.raises(L.TQError) as ei:
        fn(*args, **kw)
    assert ei.value.status == L.TQ_ERR_OVERFLOW_BIGINT, ei.value


def _key_idx(funcs, gb):
    return [i for i, (f, a) in enumerate(funcs) if f == FIRSTROW and a in gb]


def check(got, cols, gb, funcs, want=None):
    """every group's results bit-equal to the exact reference, NULL masks included"""
    want = want or R.expect(cols, gb, funcs)
    assert not want.overflow, "the data leaves int64: the aggregation must fail instead"
    bad = R.mismatches(R.result_rows(got, _key_idx(funcs, gb)), want, funcs)
    assert not bad, f"{len(bad)} wrong results (group, function, expected, got), first: {bad[:5]}"
    return want


def _funcs(nk, xc):
    return [(COUNT, -1), (COUNT, xc), (SUM, xc), (AVG, xc), (MAX, xc), (MIN, xc), (FIRSTROW, xc)] + [(FIRSTROW, g) for g in range(nk)]


def _family(name, seed):
    """(family, types, cols) with the BIGINT key of key_column: edge keys and the NULL key among the groups"""
    fam = R.check_family(R.make(name, np.random.default_rng(seed)))
    tp = UINT64 if fam.x.dtype == np.uint64 else INT64
    return fam, [INT64, tp], [R.key_column(fam.gid), Column(tp, fam.x, fam.nn)]


def _sorted_by_group(cols, gid):
    """the rows reordered into runs of one group (each group's own rows keep their order)"""
    order = np.argsort(gid, kind="stable")
    return [Column(c.tp, c.values[order], c.not_null()[order]) for c in cols]


# ------------------------------------------------------------------ the general update kernel
@pytest.mark.parametrize("family", FAMS)
def test_random_keys(lib, family):
    """k_agg_update with the family's rows interleaved at random: a warp's rows land in different slots"""
    fam, types, cols = _family(family, 1 + FAMS.index(family))
    funcs = _funcs(1, 1)
    got, _ = run_host(lib, types, cols, [0], funcs, int(fam.gid.max()) + 1)
    check(got, cols, [0], funcs)


@pytest.mark.parametrize("family", FAMS)
def test_clustered_keys(lib, family):
    """the same rows in runs of one group: most warps see one live slot, so COUNT takes the shuffle-reduced branch, while
    int SUM / AVG still add row by row into the 128-bit state"""
    fam, types, cols = _family(family, 11 + FAMS.index(family))
    cols = _sorted_by_group(cols, fam.gid)
    funcs = _funcs(1, 1)
    got, _ = run_host(lib, types, cols, [0], funcs, int(fam.gid.max()) + 1)
    check(got, cols, [0], funcs)


@pytest.mark.parametrize("twin", sorted(R.TWINS))
def test_out_by_one_twins(lib, twin):
    """the in-range `limits` dataset gives exact values; its twin, whose one group totals one past a limit (or ±2^64: the low
    word is exactly 0 there), must fail with ErrOverflow — on random and on clustered rows"""
    rng = np.random.default_rng(31)
    base = R.check_family(R.limits(rng, 180, 2, 800))
    t = R.check_family(R.out_by_one(base, R.TWINS[twin], rng))
    funcs = _funcs(1, 1)
    for fam in (base, t):
        types, cols = [INT64, INT64], [R.key_column(fam.gid), Column(INT64, fam.x)]
        for c in (cols, _sorted_by_group(cols, fam.gid)):
            if fam is base:
                check(run_host(lib, types, c, [0], funcs, 180)[0], c, [0], funcs)
            else:
                assert R.expect(c, [0], funcs).overflow
                raises_overflow(run_host, lib, types, c, [0], funcs, 180)
                raises_overflow(run_host, lib, types, c, [0], [(SUM, 1), (FIRSTROW, 0)], 180)   # SUM alone
                raises_overflow(run_host, lib, types, c, [0], [(AVG, 1), (FIRSTROW, 0)], 180)   # AVG alone


# ------------------------------------------------------------------ no GROUP BY
SCALAR_TARGETS = {"max": R.INT64_MAX, "min": R.INT64_MIN, "max_plus_1": R.INT64_MAX + 1, "min_minus_1": R.INT64_MIN - 1}


def _scalar_rows(rng, n, target):
    """n rows drawn from the limits and prefix_wraps terms, then extreme terms and one remainder that make the exact total
    `target`, shuffled"""
    pool = np.concatenate([R.limits(rng, 120, 2, 2000).x, R.prefix_wraps(rng, 100).x])
    x = rng.choice(pool, n)
    c = target - R.segment_sums(x, [0])[0]
    extra = []
    while not R.in_range(c):
        t = R.INT64_MAX if c > 0 else R.INT64_MIN
        extra.append(t)
        c -= t
    x = np.concatenate([x, np.array(extra + [c], dtype=np.int64)])
    return x[rng.permutation(len(x))]


@pytest.mark.parametrize("target", sorted(SCALAR_TARGETS))
def test_scalar_aggregate_8e6_rows(lib, target):
    """every row goes to one 128-bit state: 8e6 atomics on one low word, its carries deciding the high word"""
    rng = np.random.default_rng(41 + sorted(SCALAR_TARGETS).index(target))
    x = Column(INT64, _scalar_rows(rng, 8_000_000, SCALAR_TARGETS[target]))
    funcs = [(COUNT, -1), (COUNT, 0), (SUM, 0), (AVG, 0), (MAX, 0), (MIN, 0)]
    want = R.expect([x], [], funcs)
    assert R.segment_sums(x.values, [0])[0] == SCALAR_TARGETS[target]
    if want.overflow:
        raises_overflow(run_host, lib, [INT64], [x], [], funcs, 0, chunk=1 << 20)
    else:
        got, _ = run_host(lib, [INT64], [x], [], funcs, 0, chunk=1 << 20)
        check(got, [x], [], funcs, want)


# ------------------------------------------------------------------ the flag word
@pytest.mark.parametrize("tp", [INT64, UINT64])
def test_not_null_compact_state_then_nullable_batches(lib, tp):
    """extremes_only (MAX of INT64_MIN and MIN of UINT64_MAX leave the zero state as it was):
    (1) arguments declared NOT NULL: no flag word; (2) a nullable argument that has only seen batches without a bitmap: the
    flag word exists but is not maintained; (3) then a batch with a NULL bitmap, new groups and NULL-only groups among it:
    k_agg_set_flags back-fills the flags of the groups that exist, which must keep their extreme MAX / MIN"""
    rng = np.random.default_rng(51 + tp)
    fam = R.check_family(R.extremes_only(rng, tp, copies=8))
    k = R.key_column(fam.gid)
    first = fam.nn & k.not_null() & (fam.gid % 2 == 0)          # batch 1: no NULLs at all, half the groups
    types, funcs = [INT64, tp], _funcs(1, 1)
    b1 = [Column(INT64, k.values[first]), Column(tp, fam.x[first])]   # no bitmaps
    got, _ = run_host(lib, types, b1, [0], funcs, 64, not_null=(0, 1))
    check(got, b1, [0], funcs)
    got, _ = run_host(lib, types, b1, [0], funcs, 64)
    check(got, b1, [0], funcs)
    b2 = [Column(INT64, k.values[~first], k.not_null()[~first]), Column(tp, fam.x[~first], fam.nn[~first])]
    got, _ = run_device(lib, types, [b1, b2], [0], funcs, 64)
    allc = [Column(INT64, np.concatenate([b1[0].values, b2[0].values]), np.concatenate([np.ones(first.sum(), bool), b2[0].not_null()])),
            Column(tp, np.concatenate([b1[1].values, b2[1].values]), np.concatenate([np.ones(first.sum(), bool), b2[1].not_null()]))]
    want = check(got, allc, [0], funcs)
    assert any(v is None for r in want.groups.values() for v in r[2:6])   # NULL-only groups are part of it


# ------------------------------------------------------------------ growth
@pytest.mark.parametrize("family", ["limits", "prefix_wraps", "unsigned"])
def test_table_growth_and_deferred_replay(lib, family):
    """est_groups=1: the table starts at 2^16 slots (load limit 32,768).  Batch 1 holds the first part of every family
    group's rows (prefix_wraps: all but the last, so every state is out of int64; the other families: the first half, some
    states out of int64), so the 128-bit states are mid-sum when batch 2 brings 100,000 new groups: rows are deferred,
    k_agg_rehash moves the mid-sum states and the deferred rows are replayed within that put.  Batch 3 brings the rest of the
    family's rows to the moved states."""
    fam, types, cols = _family(family, 61 + FAMS.index(family))
    rng = np.random.default_rng(7)
    order = np.argsort(fam.gid, kind="stable")
    pos = np.empty(len(order), np.int64)
    pos[order] = np.arange(len(order)) - np.searchsorted(fam.gid[order], fam.gid[order])   # position inside the group
    size = np.bincount(fam.gid)[fam.gid]
    early = pos < np.maximum(size - 1, 1) if family == "prefix_wraps" else pos < size // 2
    nf = 300_000
    fk = Column(INT64, (np.int64(1) << 40) + rng.integers(0, 100_000, nf))
    assert not np.intersect1d(fk.values, cols[0].values).size
    b1 = [Column(c.tp, c.values[early], c.not_null()[early]) for c in cols]
    b2 = [fk, Column(cols[1].tp, rng.integers(0, 1 << 20, nf).astype(cols[1].values.dtype))]
    b3 = [Column(c.tp, c.values[~early], c.not_null()[~early]) for c in cols]
    mid = [not R.in_range(t) for t in R.group_sums(fam.gid[early], b1[1].values, b1[1].not_null())]
    assert all(mid) if family == "prefix_wraps" else any(mid), "batch 1 leaves no state outside int64"
    funcs = _funcs(1, 1)
    launches = []
    got, _ = run_device(lib, types, [b1, b2, b3], [0], funcs, 1, launches=launches)
    allc = [Column(types[i], np.concatenate([b[i].values for b in (b1, b2, b3)]), np.concatenate([b[i].not_null() for b in (b1, b2, b3)]))
            for i in range(2)]
    check(got, allc, [0], funcs)
    # batch 2 = the first update round, the growth, then at least one replay round: the rehash ran between batches 1 and 3
    assert launches[1] - launches[0] >= 2, f"update launches per put {launches}: batch 2 did not grow the table"


# ------------------------------------------------------------------ other key encodings
def test_multi_column_and_varchar_group_by(lib):
    """one limits dataset under a two-column GROUP BY (MultiKeyEncoder, dict.cu) and under a VARCHAR GROUP BY (dictionary
    ids, strdict.cu); the key tuples / strings name the same groups as the BIGINT key"""
    fam, types, cols = _family("limits", 71)
    g = fam.gid
    k2 = Column(UINT64, (g.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(1 << 63), g % 7 != 3)
    t2, c2 = [INT64, UINT64, INT64], [cols[0], k2, cols[1]]
    funcs = _funcs(2, 2)
    got, _ = run_host(lib, t2, c2, [0, 1], funcs, 400)
    check(got, c2, [0, 1], funcs)
    s = Column(BYTES, [None if v == 5 else b"grp-%05d" % v for v in g.tolist()])
    t3, c3 = [BYTES, INT64], [s, cols[1]]
    funcs = _funcs(1, 1)
    got, _ = run_host(lib, t3, c3, [0], funcs, 400)
    check(got, c3, [0], funcs)


@pytest.mark.parametrize("family", FAMS)
def test_device_memory_input(lib, family):
    """three TQ_MEM_DEVICE batches"""
    fam, types, cols = _family(family, 81 + FAMS.index(family))
    n = cols[0].length
    cuts = [0, n // 3, 2 * n // 3, n]
    batches = [[c.slice(lo, hi) for c in cols] for lo, hi in zip(cuts[:-1], cuts[1:])]
    funcs = _funcs(1, 1)
    got, _ = run_device(lib, types, batches, [0], funcs, int(fam.gid.max()) + 1)
    check(got, cols, [0], funcs)


# ------------------------------------------------------------------ partial rows
def _two_part_groups(rng, n_groups, past=None):
    """groups whose rows split into two parts: part totals a and b in int64, a + b at INT64_MAX or INT64_MIN.
    past='merged': group 0's a + b is INT64_MAX + 1 (both parts in range); past='part': group 0's first part totals
    INT64_MAX + 1 (the merged total is back in range).  Returns (gid, x) per part and the merged targets"""
    parts = ([], [])
    targets = []
    for g in range(n_groups):
        T = R.INT64_MAX if g % 2 == 0 else R.INT64_MIN
        a = T // 2 + int(rng.integers(-(1 << 60), 1 << 60))
        if g == 0 and past == "merged":
            T = R.INT64_MAX + 1
            a = T // 2 + 12345
        b = T - a
        if g == 0 and past == "part":
            a, b = R.INT64_MAX + 1, -5
            T = a + b
        targets.append(T)
        for p, tot in zip(parts, (a, b)):
            m = int(rng.integers(2, 300))
            if R.in_range(tot):
                p.append(R.group_terms(rng, m, tot))
            else:   # a part whose own total leaves int64: terms totalling tot - INT64_MAX, then INT64_MAX
                p.append(R.group_terms(rng, m, tot - R.INT64_MAX) + [R.INT64_MAX])
    out = []
    for p in parts:
        gid, vals = R.interleave(rng, p)
        out.append((gid, vals.astype(np.int64)))
    return out, targets


EM_CASES = ["in_range", "merged_past", "part_past"]


@pytest.mark.parametrize("case", EM_CASES)
def test_export_and_merge(lib, case):
    """two Partial1 handles export (tq_agg_export_partial) and a third merges them (tq_agg_merge_partial): merged totals at
    INT64_MAX / INT64_MIN are exact; a merged total one past the limit fails in the merging handle; a part whose own total
    leaves int64 fails in its export, as the reference's Partial1 worker does"""
    rng = np.random.default_rng(91 + EM_CASES.index(case))
    parts, targets = _two_part_groups(rng, 60, {"in_range": None, "merged_past": "merged", "part_past": "part"}[case])
    types, funcs = [INT64, INT64], _funcs(1, 1)
    pcols = [[R.key_column(gid), Column(INT64, x)] for gid, x in parts]
    allc = [Column(INT64, np.concatenate([p[0].values for p in pcols]), np.concatenate([p[0].not_null() for p in pcols])),
            Column(INT64, np.concatenate([p[1].values for p in pcols]))]
    want = R.expect(allc, [0], funcs)
    if case == "in_range":
        got = run_export_merge(lib, types, pcols, [0], funcs, 64)
        check(got, allc, [0], funcs, want)
        assert {r[2] for r in want.groups.values()} == {R.INT64_MAX, R.INT64_MIN}
    elif case == "merged_past":
        assert want.overflow and not any(R.expect(p, [0], funcs).overflow for p in pcols)
        raises_overflow(run_export_merge, lib, types, pcols, [0], funcs, 64)
    else:
        assert not want.overflow and R.expect(pcols[0], [0], funcs).overflow
        raises_overflow(run_export_merge, lib, types, pcols, [0], funcs, 64)
        raises_overflow(run_export_merge, lib, types, pcols[:1], [0], [(SUM, 1), (FIRSTROW, 0)], 64)


FINAL_CASES = ["limits", "past"]


@pytest.mark.parametrize("tp", [INT64, UINT64])
@pytest.mark.parametrize("case", FINAL_CASES)
def test_final_mode(lib, case, tp):
    """FinalMode (tq_agg_create_final) over partial rows built by the exact reference (the oracle's Partial1 raises on prefix
    overflow): two regions whose totals are in range, merged at INT64_MAX / INT64_MIN, or one past INT64_MAX; and extra
    partial rows with a NULL SUM and an AVG (count, NULL) pair, which must be skipped count included"""
    rng = np.random.default_rng(101 + FINAL_CASES.index(case) + 7 * tp)
    parts, _ = _two_part_groups(rng, 40, None if case == "limits" else "merged")
    funcs = [(COUNT, 1), (SUM, 1), (AVG, 1), (MAX, 1), (MIN, 1), (FIRSTROW, 1), (FIRSTROW, 0)]
    types = [INT64, tp]
    chunks, ptypes = [], None
    for gid, x in parts:
        ptypes, ch = R.expect_partial(types, [R.key_column(gid), Column(tp, x.view(np.uint64) if tp == UINT64 else x)], [0], funcs)
        chunks.append(ch)
    ng = int(parts[0][0].max()) + 1
    # per group one more partial row: COUNT 3, SUM NULL, AVG (5, NULL), MAX / MIN / FIRSTROW(x) NULL, then the key twice
    keys = R.key_column(np.arange(ng)).tolist()
    extra = [R.column(INT64, [3] * ng), R.column(INT64, [None] * ng), R.column(INT64, [5] * ng), R.column(INT64, [None] * ng),
             R.column(tp, [None] * ng), R.column(tp, [None] * ng), R.column(tp, [None] * ng), R.column(INT64, keys), R.column(INT64, keys)]
    assert len(extra) == len(ptypes)
    pcols = [Column(t, np.concatenate([ch.cols[c].values for ch in chunks] + [extra[c].values]),
                    np.concatenate([ch.cols[c].not_null() for ch in chunks] + [extra[c].not_null()])) for c, t in enumerate(ptypes)]
    ff, pgb = R.final_funcs(funcs, 1)
    want = R.expect_final(pcols, pgb, ff)
    ffuncs = [(f, a) for f, a, _ in ff]
    if case == "past":
        assert want.overflow
        raises_overflow(run_final, ptypes, pcols, pgb, ff)
        return
    got = run_final(ptypes, pcols, pgb, ff)
    key_out = [len(funcs) - 1]   # FIRSTROW(key) reads its own partial column
    assert not want.overflow
    bad = R.mismatches(R.result_rows(got, key_out), want, ffuncs)
    assert not bad, bad[:5]
    assert {r[1] for r in want.groups.values()} == {R.INT64_MAX, R.INT64_MIN}


# ------------------------------------------------------------------ pre-aggregation
def test_preaggregation_decision(lib, monkeypatch):
    """a NOT NULL batch of 2^20+ rows over the 360 groups of a limits dataset (its zero-total groups' rows repeated until the
    batch is large enough, which leaves every total as it was): a handle with an int SUM stays on the general path
    (agg_try_preagg covers COUNT and DOUBLE SUM / AVG only), so its launch count equals that of TQ_AGG_NO_PREAGG=1; the same
    handle without the SUM takes k_agg_preagg (one launch more), counts exact"""
    rng = np.random.default_rng(111)
    fam = R.check_family(R.limits(rng, 360, 2, 2000))
    zero = np.isin(fam.gid, [g for g, t in enumerate(fam.meta["targets"]) if t == 0])
    copies = -(-((1 << 20) + 50_000 - len(fam.gid)) // int(zero.sum()))
    gid = np.concatenate([fam.gid] + [fam.gid[zero]] * copies)
    xv = np.concatenate([fam.x] + [fam.x[zero]] * copies)
    perm = rng.permutation(len(gid))
    k, x = Column(INT64, gid[perm].astype(np.int64) * 7919 + 17), Column(INT64, xv[perm])
    assert x.length >= (1 << 20) and R.group_totals(R.Family("", gid, xv, np.ones(len(gid), bool), {})) == fam.meta["targets"]
    types, cols = [INT64, INT64], [k, x]
    for funcs in ([(COUNT, -1), (COUNT, 1), (SUM, 1), (FIRSTROW, 0)], [(COUNT, -1), (COUNT, 1), (FIRSTROW, 0)]):
        want = R.expect(cols, [0], funcs)
        launches = {}
        for env in ({"TQ_AGG_NO_PREAGG": "1"}, {}):
            _switches(monkeypatch, env)
            got, st = run_host(lib, types, cols, [0], funcs, 360, not_null=(0, 1), chunk=1 << 20)
            check(got, cols, [0], funcs, want)
            launches[bool(env)] = st[3]
        _switches(monkeypatch, {})
        if len(funcs) > 3:
            assert launches[False] == launches[True], f"the int SUM handle left the general path: {launches}"
        else:
            assert launches[False] == launches[True] + 1, f"the COUNT-only handle did not pre-aggregate: {launches}"
