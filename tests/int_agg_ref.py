"""Exact per-group BIGINT / BIGINT UNSIGNED aggregation on Python ints, and datasets aimed at the int64 limits (TEST
INFRASTRUCTURE).

The device keeps an int SUM / AVG as an exact 128-bit sum and reports ErrOverflow iff a group's exact total leaves int64,
whatever the order of its rows (DESIGN §3 deviation i).  The C oracle adds in row order and raises on the first prefix that
leaves int64 (types.AddInt64), so it cannot be the yardstick where the two differ.  This module is:

  SUM       the exact total; an error iff some group's total leaves [-2^63, 2^63)
  AVG       trunc(total / count), rounding toward zero as Go's integer division does (-7 / 2 = -3)
  COUNT     exact
  MAX / MIN signed order for BIGINT, unsigned order for BIGINT UNSIGNED
  FIRSTROW  of a non-key column: the set of the group's values, None for a NULL row (any row may claim a group: deviation ii)
  a BIGINT UNSIGNED argument of SUM / AVG is read as int64 (sum4Int64 reads EvalInt, func_sum.go:118), so 2^63 adds -2^63

Groups follow HashGroupKey (float_agg_ref.group_rows): NULL is its own group, integer keys compare bitwise.

Exact sums are vectorised by splitting each int64 into a signed high half and an unsigned low half (32 bits each): both
halves sum exactly in int64 for fewer than 2^31 rows per group."""
from collections import namedtuple

import numpy as np

from float_agg_ref import group_rows, key_labels
from hash_targets import EMPTY_KEY
from tinysql_b200.chunk import INT64, UINT64, Chunk, Column

COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
UINT64_MAX = (1 << 64) - 1
TWO62 = 1 << 62
EMPTY_KEY_I64 = EMPTY_KEY - (1 << 64)   # the aggregation table's free-slot marker as a BIGINT key: it lives in a side slot
EDGE_KEYS = [INT64_MIN, INT64_MAX, -1, 0, EMPTY_KEY_I64]   # plus NULL
TARGETS = [INT64_MAX, INT64_MIN, 0, -1, 1, TWO62, -TWO62, INT64_MAX - 1, INT64_MIN + 1]


def as_i64(v):
    """the signed reading of a Python int in [-2^63, 2^64)"""
    return v - (1 << 64) if v > INT64_MAX else v


def in_range(t):
    return INT64_MIN <= t <= INT64_MAX


def trunc_div(a, b):
    """Go's a / b on integers: the quotient rounded toward zero"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


# ------------------------------------------------------------------ exact sums
def _split(x):
    x = np.asarray(x).view(np.int64) if np.asarray(x).dtype == np.uint64 else np.asarray(x, dtype=np.int64)
    return x >> 32, x & 0xFFFFFFFF


def _join(hi, lo):
    return [(int(h) << 32) + int(l) for h, l in zip(hi, lo)]


def segment_sums(x, starts):
    """exact int sums (Python ints) of x[starts[i]:starts[i+1]] (the last segment runs to the end); empty segments sum to 0"""
    hi, lo = _split(x)
    n = len(hi)
    starts = np.asarray(starts, dtype=np.int64)
    if n == 0:
        return [0] * len(starts)
    ends = np.append(starts[1:], n)
    ch, cl = np.concatenate([[0], np.cumsum(hi)]), np.concatenate([[0], np.cumsum(lo)])
    return _join(ch[ends] - ch[starts], cl[ends] - cl[starts])


def prefix_out_of_range(x):
    """bool per position k: does the in-order sum x[0..k] leave int64 (exact, vectorised)"""
    hi, lo = _split(x)
    h, l = np.cumsum(hi), np.cumsum(lo)
    h = h + (l >> 32)   # normalise: the prefix = h * 2^32 + (l mod 2^32) with the low part in [0, 2^32)
    return (h >= (1 << 31)) | (h < -(1 << 31))


# ------------------------------------------------------------------ the reference
Expected = namedtuple("Expected", "groups overflow")
"""groups: {group key tuple: [per function: int, None (= NULL) or, for FIRSTROW of a non-key column, a frozenset]};
overflow: some group's SUM / AVG total leaves int64 (the aggregation must fail with ErrOverflow)"""


def _grouped(gid, n_groups, sel):
    """(row order sorted by group among rows `sel`, start of each group in that order)"""
    rows = np.nonzero(sel)[0]
    order = rows[np.argsort(gid[rows], kind="stable")]
    return order, np.searchsorted(gid[order], np.arange(n_groups))


def expect(cols, group_by, funcs):
    """the exact result of HashAgg(group_by; funcs) over BIGINT / BIGINT UNSIGNED arguments (keys of any type)"""
    n = cols[0].length if cols else 0
    gid, labels = group_rows([cols[g] for g in group_by], n)
    ng = len(labels)
    rows = [[None] * len(funcs) for _ in range(ng)]
    overflow = False
    for fi, (f, a) in enumerate(funcs):
        if a < 0:
            nn, x = np.ones(n, bool), np.ones(n, np.int64)
        else:
            nn, x = cols[a].not_null(), cols[a].values
        order, starts = _grouped(gid, ng, nn)
        cnt = np.diff(np.append(starts, len(order)))
        if f == COUNT:
            for g in range(ng):
                rows[g][fi] = int(cnt[g])
        elif f in (SUM, AVG):
            sums = segment_sums(x[order], starts)
            for g in range(ng):
                if cnt[g] == 0:
                    continue
                overflow |= not in_range(sums[g])
                rows[g][fi] = sums[g] if f == SUM else trunc_div(sums[g], int(cnt[g]))
        elif f in (MAX, MIN):
            v = x[order]
            for g in range(ng):
                if cnt[g]:
                    seg = v[starts[g]:starts[g] + cnt[g]]
                    rows[g][fi] = int(seg.max() if f == MAX else seg.min())
        else:
            if a in group_by and len(group_by) == 1:
                for g in range(ng):
                    rows[g][fi] = labels[g][0]
                continue
            vals = cols[a].tolist()
            sets = [set() for _ in range(ng)]
            for g, v in zip(gid.tolist(), vals):
                sets[g].add(v)
            for g in range(ng):
                rows[g][fi] = frozenset(sets[g])
    return Expected({lab: r for lab, r in zip(labels, rows)}, overflow)


def result_rows(chunk, key_idx):
    """{group key tuple: [per result column: int or None]} of a device / oracle result; key_idx: its FIRSTROW(key) columns.
    No group may appear twice."""
    keys = list(zip(*[key_labels(chunk.cols[c]) for c in key_idx])) if key_idx else [()] * chunk.num_rows()
    vals = [c.tolist() for c in chunk.cols]
    out = {k: [v[i] for v in vals] for i, k in enumerate(keys)}
    assert len(out) == len(keys), "two result rows for one group"
    return out


def mismatches(got, want, funcs):
    """the (group, function, expected, got) of every result that is not bit-equal to the reference (FIRSTROW: a member of
    the group's set), and of every group missing or extra"""
    bad = [(k, None, "missing group", None) for k in want.groups if k not in got]
    bad += [(k, None, "extra group", None) for k in got if k not in want.groups]
    for k, w in want.groups.items():
        if k not in got:
            continue
        for fi, wv in enumerate(w):
            gv = got[k][fi]
            ok = gv in wv if isinstance(wv, frozenset) else (gv == wv and (gv is None) == (wv is None))
            if not ok:
                bad.append((k, fi, wv if not isinstance(wv, frozenset) or len(wv) < 6 else f"one of {len(wv)} values", gv))
    return bad


def expect_partial(types, cols, group_by, funcs):
    """one region's Partial1 rows in the coprocessor's layout (store/mockstore/mocktikv/aggregate.go:81-124): per function its
    partial columns — COUNT: count; SUM: total (NULL for no input); AVG: (count, total); MAX / MIN / FIRSTROW: value — then the
    GROUP BY columns.  FIRSTROW takes the region's first row of the group.  Returns (types, Chunk); raises OverflowError if
    a total leaves int64, as the reference's Partial1 worker does."""
    n = cols[0].length
    gid, labels = group_rows([cols[g] for g in group_by], n)
    first = np.zeros(len(labels), np.int64)
    first[gid[::-1]] = np.arange(n)[::-1]
    inner = []   # the functions whose results make up the partial columns
    for f, a in funcs:
        inner += [(COUNT, a), (SUM, a)] if f == AVG else ([] if f == FIRSTROW else [(f, a)])
    want = expect(cols, group_by, inner)
    if want.overflow:
        raise OverflowError("a partial total leaves int64")
    res = [want.groups[lab] for lab in labels]
    out_t, out_v, i = [], [], 0
    for f, a in funcs:
        if f == FIRSTROW:
            v = cols[a].tolist()
            out_t.append(types[a]); out_v.append([v[r] for r in first])
            continue
        for _ in range(2 if f == AVG else 1):
            out_t.append(types[a] if f in (MAX, MIN) else INT64); out_v.append([r[i] for r in res])
            i += 1
    for g in group_by:
        v = cols[g].tolist()
        out_t.append(types[g]); out_v.append([v[r] for r in first])
    return out_t, Chunk([column(t, v) for t, v in zip(out_t, out_v)])


def expect_final(pcols, group_by, ffuncs):
    """FinalMode over partial rows, ffuncs = [(func, arg_col, arg_col2)]: COUNT adds the partial counts; SUM adds the non-NULL
    partial totals; AVG adds (count, total) over the rows whose count and total are both non-NULL (func_avg.go:96-110);
    MAX / MIN over the non-NULL partials (unsigned order for a BIGINT UNSIGNED column); FIRSTROW: the set of the partial
    values.  Partial totals of a BIGINT UNSIGNED column are read as int64."""
    gid, labels = group_rows([pcols[g] for g in group_by], pcols[0].length if pcols else 0)
    vals = [c.tolist() for c in pcols]
    acc = [[None] * len(ffuncs) for _ in labels]
    cnt = [[0] * len(ffuncs) for _ in labels]
    for r, g in enumerate(gid.tolist()):
        for fi, (f, a, b) in enumerate(ffuncs):
            v, cur = vals[a][r], acc[g][fi]
            if f == FIRSTROW:
                acc[g][fi] = (cur or frozenset()) | {v}
            elif f == AVG:
                s = vals[b][r]
                if v is not None and s is not None:
                    cnt[g][fi] += v
                    acc[g][fi] = (cur or 0) + as_i64(s)
            elif v is None:
                continue
            elif f in (COUNT, SUM):
                acc[g][fi] = (cur or 0) + (v if f == COUNT else as_i64(v))
            else:
                acc[g][fi] = v if cur is None else (max(cur, v) if f == MAX else min(cur, v))
    overflow = False
    for g in range(len(labels)):
        for fi, (f, a, b) in enumerate(ffuncs):
            if f == COUNT:
                acc[g][fi] = acc[g][fi] or 0
            elif f == SUM and acc[g][fi] is not None:
                overflow |= not in_range(acc[g][fi])
            elif f == AVG:
                if cnt[g][fi] == 0:
                    acc[g][fi] = None
                else:
                    overflow |= not in_range(acc[g][fi])
                    acc[g][fi] = trunc_div(acc[g][fi], cnt[g][fi])
    return Expected({lab: r for lab, r in zip(labels, acc)}, overflow)


def final_funcs(funcs, n_group_by):
    """the FinalMode descriptors (func, arg_col, arg_col2) over the partial rows of expect_partial: partial columns in function
    order (AVG: count, then total), then the GROUP BY columns, whose indices are returned second"""
    out, c = [], 0
    for f, _ in funcs:
        out.append((f, c, c + 1) if f == AVG else (f, c, -1))
        c += 2 if f == AVG else 1
    return out, list(range(c, c + n_group_by))


def column(tp, vals):
    """a Column of Python ints / None (BIGINT UNSIGNED values in [0, 2^64))"""
    nn = [v is not None for v in vals]
    dt = np.uint64 if tp == UINT64 else np.int64
    arr = np.array([0 if v is None else v for v in vals], dtype=object).astype(dt) if vals else np.zeros(0, dt)
    return Column(tp, arr, nn)


# ------------------------------------------------------------------ aimed data
Family = namedtuple("Family", "name gid x nn meta")
"""gid: group id per row (int64 >= 0, ids 0..len(EDGE_KEYS) map to the edge keys, see key_column); x: the argument
(np.int64, np.uint64 for the unsigned family); nn: its NOT NULL mask; meta: what the family aims at, for its self-check"""
FAMILIES = ("limits", "prefix_wraps", "unsigned", "avg_trunc", "extremes_only")


def _random63(rng):
    return int(rng.integers(0, 1 << 63, dtype=np.uint64)) * (1 if rng.random() < 0.5 else -1)


LIMIT_POOL = [INT64_MIN, INT64_MAX, TWO62, -TWO62, -INT64_MAX]


def group_terms(rng, m, target, pool=LIMIT_POOL, p_random=0.3):
    """m int64 terms that sum exactly to `target`: m - 1 drawn from `pool` or random 63-bit values of either sign, each
    kept so that the running distance to the target stays inside int64, then one last term that lands on the target"""
    terms, s = [], 0
    while len(terms) < m - 1:
        t = _random63(rng) if rng.random() < p_random else pool[int(rng.integers(len(pool)))]
        if not in_range(target - s - t):   # the term that would close the group here must be an int64
            continue
        terms.append(t)
        s += t
    terms.append(target - s)
    assert in_range(terms[-1])
    return terms


def interleave(rng, per_group):
    """rows of several groups mixed at random, each group's own rows kept in their order: (gid, values)"""
    gid = np.repeat(np.arange(len(per_group)), [len(t) for t in per_group])
    gid = gid[rng.permutation(len(gid))]
    pos = np.zeros(len(per_group), np.int64)
    vals = np.empty(len(gid), dtype=object)
    for i, g in enumerate(gid.tolist()):
        vals[i] = per_group[g][pos[g]]
        pos[g] += 1
    return gid, vals


def _sizes(rng, n_groups, lo, hi):
    """group sizes spread log-uniformly over [lo, hi], both ends included"""
    s = np.exp(rng.uniform(np.log(lo), np.log(hi + 1), n_groups)).astype(np.int64)
    s[:2] = [lo, hi]
    return np.clip(s, lo, hi)


def limits(rng, n_groups=360, lo=2, hi=2000):
    """groups of lo..hi terms from {INT64_MIN, INT64_MAX, ±2^62, -(2^63 - 1), random 63-bit}, both signs; group g's total is
    TARGETS[g % 9]"""
    sizes = _sizes(rng, n_groups, lo, hi)
    targets = [TARGETS[g % len(TARGETS)] for g in range(n_groups)]
    terms = [group_terms(rng, int(m), t) for m, t in zip(sizes, targets)]
    gid, vals = interleave(rng, terms)
    return Family("limits", gid, vals.astype(np.int64), np.ones(len(gid), bool), {"targets": targets, "sizes": (lo, hi)})


def out_by_one(fam, want_total, rng):
    """the twin of a `limits` family that differs only in the terms of one group, whose total becomes want_total (one past
    an int64 limit, or ±2^64); the group is one with at least 4 terms whose target is nearest"""
    targets = fam.meta["targets"]
    sizes = np.bincount(fam.gid, minlength=len(targets))
    cand = [g for g in range(len(targets)) if sizes[g] >= 4]
    g = min(cand, key=lambda g: (abs(want_total - targets[g]), -sizes[g]))
    delta = want_total - targets[g]
    x = fam.x.copy()
    for r in np.nonzero(fam.gid == g)[0]:
        v = int(x[r])
        step = max(min(delta, INT64_MAX - v), INT64_MIN - v)
        x[r] = v + step
        delta -= step
        if delta == 0:
            break
    assert delta == 0
    t = list(targets)
    t[g] = want_total
    return Family(f"out_by_one[{want_total:#x}]", fam.gid, x, fam.nn, {"targets": t, "group": g})


TWINS = {"max_plus_1": INT64_MAX + 1, "min_minus_1": INT64_MIN - 1, "plus_2_64": 1 << 64, "minus_2_64": -(1 << 64)}


def prefix_wraps(rng, n_groups=300, lo=3, hi=200):
    """totals in range, but every in-order prefix of 2 .. m - 1 rows of a group leaves int64: the prefixes walk in a band
    above INT64_MAX (below INT64_MIN for the mirrored groups) and the last term brings the total back"""
    terms = []
    targets = []
    for g, m in enumerate(_sizes(rng, n_groups, lo, hi)):
        sign = 1 if g % 2 == 0 else -1
        target = int(rng.integers(TWO62, INT64_MAX))   # the last term target - prefix must reach down into int64
        band_lo, band_hi = (1 << 63) + 1, target + (1 << 63)  # prefixes 2 .. m - 1 stay in [band_lo, band_hi]
        p = [int(rng.integers(band_lo, band_hi, dtype=np.uint64)) for _ in range(int(m) - 2)]
        first = int(rng.integers(TWO62, INT64_MAX))
        while not in_range(p[0] - first):
            first = int(rng.integers(TWO62, INT64_MAX))
        seq = [first] + [b - a for a, b in zip([first] + p[:-1], p)] + [target - p[-1]]
        terms.append([sign * t for t in seq])
        targets.append(sign * target)
    gid, vals = interleave(rng, terms)
    return Family("prefix_wraps", gid, vals.astype(np.int64), np.ones(len(gid), bool), {"targets": targets})


UNSIGNED_POOL = [(1 << 63) - 1, 1 << 63, (1 << 63) + 1, UINT64_MAX, 0, 1]


def unsigned(rng, n_groups=240, lo=2, hi=400):
    """BIGINT UNSIGNED values around 2^63 - 1, 2^63, 2^63 + 1 and 2^64 - 1; read as int64 each group's total is a target;
    every group of 4 or more holds values on both sides of 2^63, so the unsigned and the signed order disagree about MAX / MIN"""
    pool = [as_i64(v) for v in UNSIGNED_POOL]
    sizes = _sizes(rng, n_groups, lo, hi)
    targets = [TARGETS[g % len(TARGETS)] for g in range(n_groups)]
    terms = []
    for m, t in zip(sizes, targets):
        while True:
            tt = group_terms(rng, int(m), t, pool, p_random=0.2)
            if m < 4 or min(tt) < 0 <= max(tt):   # below and at / above 2^63 when read unsigned
                break
        k = int(rng.integers(0, 1 + len(tt) // 8))   # NULL rows among them, whose slots hold 2^63 (ignored by every function)
        for pos in rng.integers(0, len(tt) + 1, k):
            tt.insert(int(pos), None)
        terms.append(tt)
    gid, vals = interleave(rng, terms)
    nn = np.array([v is not None for v in vals])
    x = np.where(nn, vals, INT64_MIN).astype(np.int64)
    return Family("unsigned", gid, x.view(np.uint64), nn, {"targets": targets})


def group_sums(gid, x, nn=None):
    """exact totals (Python ints) of the non-NULL rows of x per group id 0 .. max(gid)"""
    nn = np.ones(len(gid), bool) if nn is None else np.asarray(nn, dtype=bool)
    order, starts = _grouped(gid, int(gid.max()) + 1, nn)
    return segment_sums(np.asarray(x)[order], starts)


AVG_COUNTS = (2, 3, 7)


def avg_trunc(rng):
    """groups of 2, 3 and 7 rows whose totals those counts do not divide, negative and positive (small and near the limits),
    and groups totalling INT64_MIN of 1, 2 and 3 rows"""
    specs = []
    for c in AVG_COUNTS:
        for base in (7, 1000003, INT64_MAX - 10, TWO62 + 5):
            for sign in (1, -1):
                t = sign * base
                while t % c == 0:
                    t -= sign
                specs.append((c, t))
    specs += [(c, INT64_MIN) for c in (1, 2, 3)]
    terms = [group_terms(rng, c, t) for c, t in specs]
    gid, vals = interleave(rng, terms)
    return Family("avg_trunc", gid, vals.astype(np.int64), np.ones(len(gid), bool), {"specs": specs})


EXTREMES = {INT64: [INT64_MIN, INT64_MAX, -1, 0], UINT64: [0, (1 << 63) - 1, 1 << 63, UINT64_MAX]}


def extremes_only(rng, tp=INT64, copies=6):
    """groups whose every value is one extreme, with and without NULL rows, and groups of NULL rows only.  A group of an
    extreme of magnitude >= 2^62 (read as int64) holds one non-NULL value, so that its SUM stays in range; the others up to 40"""
    per, vals_of = [], []
    for v in EXTREMES[tp]:
        big = abs(as_i64(v)) >= TWO62
        for c in range(copies):
            k = 1 if big else int(rng.integers(1, 41))
            nulls = 0 if c % 2 == 0 else int(rng.integers(1, 6))
            per.append([v] * k + [None] * nulls)
            vals_of.append(v)
    for c in range(copies):
        per.append([None] * int(rng.integers(1, 8)))
        vals_of.append(None)
    per = [list(np.array(p, dtype=object)[rng.permutation(len(p))]) for p in per]
    gid, vals = interleave(rng, per)
    nn = np.array([v is not None for v in vals])
    dt = np.uint64 if tp == UINT64 else np.int64
    x = np.array([0 if v is None else v for v in vals], dtype=object).astype(dt)
    return Family("extremes_only", gid, x, nn, {"values": vals_of, "tp": tp})


def make(name, rng):
    return {"limits": limits, "prefix_wraps": prefix_wraps, "unsigned": unsigned, "avg_trunc": avg_trunc,
            "extremes_only": extremes_only}[name](rng)


def key_column(gid, spread=True):
    """the BIGINT GROUP BY column of group ids: ids 0..4 take the edge keys INT64_MIN, INT64_MAX, -1, 0 and the table's
    free-slot marker, id 5 is the NULL key, the others become distinct keys (spread over the 64-bit range when `spread`)"""
    ng = int(gid.max()) + 1 if len(gid) else 0
    rest = np.arange(ng - 6, dtype=np.int64) * 7919 + 17
    if spread:
        rest = rest * np.int64(0x9E3779B97F4A7C1)   # wraps: odd multiples spread over the range, still distinct
    keys = np.concatenate([np.array(EDGE_KEYS, np.int64), [0], rest])[:ng]
    nn = gid != 5
    return Column(INT64, keys[gid], nn)


# ------------------------------------------------------------------ self-checks: each family reaches its target
def group_totals(fam):
    return group_sums(fam.gid, fam.x, fam.nn)


def _carries(x):
    """how many times the unsigned low word wraps when x is added in order"""
    u = np.asarray(x).view(np.uint64)
    lo = np.cumsum(u)   # modulo 2^64
    prev = np.concatenate([[np.uint64(0)], lo[:-1]])
    return int(np.count_nonzero(lo < prev))


def check_family(fam):
    """assert that the family's data is aimed where its name says; returns fam"""
    ng = int(fam.gid.max()) + 1
    sizes = np.bincount(fam.gid, minlength=ng)
    name = fam.name.split("[")[0]
    if name in ("limits", "out_by_one", "prefix_wraps", "unsigned"):
        tot = group_totals(fam)
        assert tot == list(fam.meta["targets"]), "a group misses its target total"
    if name == "limits":
        assert set(fam.meta["targets"]) == set(TARGETS)
        assert (sizes.min(), sizes.max()) == fam.meta["sizes"]
        x = fam.x
        for g in range(ng):
            seg = x[fam.gid == g]
            if len(seg) >= 8:
                assert (seg < 0).any() and (seg > 0).any(), "a group without both signs"
            if len(seg) >= 64:   # the low word wraps many times, in either direction
                with np.errstate(over="ignore"):
                    assert _carries(seg) >= len(seg) // 8, g
        for v in (INT64_MIN, INT64_MAX, TWO62, -TWO62):
            assert (x == v).any()
    if name == "out_by_one":
        g = fam.meta["group"]
        assert not in_range(fam.meta["targets"][g])
        assert sum(not in_range(t) for t in fam.meta["targets"]) == 1
    if name == "prefix_wraps":
        order = np.argsort(fam.gid, kind="stable")
        starts = np.searchsorted(fam.gid[order], np.arange(ng))
        for g in range(ng):
            seg = fam.x[order[starts[g]:starts[g] + sizes[g]]]
            out = prefix_out_of_range(seg)
            assert out[1:-1].all() and not out[-1] and len(seg) >= 3, g
    if name == "unsigned":
        u = fam.x
        for v in UNSIGNED_POOL[:4]:
            assert (u == np.uint64(v)).any(), v
        assert all(in_range(t) for t in fam.meta["targets"])
        for g in range(ng):
            seg = u[(fam.gid == g) & fam.nn]
            if len(seg) >= 2 and (seg >= np.uint64(1 << 63)).any() and (seg < np.uint64(1 << 63)).any():
                break
        else:
            raise AssertionError("no group where the unsigned and the signed order disagree")
    if name == "avg_trunc":
        tot = group_totals(fam)
        specs = fam.meta["specs"]
        assert [t for _, t in specs] == tot and [c for c, _ in specs] == sizes.tolist()
        neg = [(c, t) for c, t in specs if t < 0 and t % c]
        pos = [(c, t) for c, t in specs if t > 0 and t % c]
        assert {c for c, _ in neg} == {c for c, _ in pos} == set(AVG_COUNTS)
        assert all(trunc_div(t, c) != t // c for c, t in neg)   # toward zero and toward -inf differ on every negative one
        assert {c for c, t in specs if t == INT64_MIN} == {1, 2, 3}
    if name == "extremes_only":
        vals_of = fam.meta["values"]
        for g in range(ng):
            seg = fam.x[(fam.gid == g) & fam.nn]
            if vals_of[g] is None:
                assert len(seg) == 0
            else:
                assert len(seg) >= 1 and (seg == seg.dtype.type(vals_of[g])).all()
        assert set(v for v in vals_of if v is not None) == set(EXTREMES[fam.meta["tp"]])
        assert any(not fam.nn[fam.gid == g].all() for g in range(ng) if vals_of[g] is not None)
    return fam
