"""GPU suite: GROUP BY over the region exchange (tq_agg_push_partial -> tq_region_wait -> tq_agg_merge_regions) with W ranks
emulated in one process (tests/exchange_ref.py's Regions layout: every rank's regions in this GPU's memory, guarded by
sentinels).  The union of the ranks' results must equal oracle_py.hash_agg over every shard, and every group must be
finished exactly once, on the rank tests/region_agg_ref.py's twin of the destination rule names."""
import ctypes as C

import numpy as np
import pytest

import exchange_ref as X
import region_agg_ref as RA
import region_outer_ref as R
from tinysql_b200 import _lib as L

pytestmark = pytest.mark.gpu

COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)
I64, U64, F64 = L.TQ_TYPE_INT64, L.TQ_TYPE_UINT64, L.TQ_TYPE_FLOAT64
WS = [1, 2, 3, 8]


@pytest.fixture(scope="module")
def lib():
    lib = L.load()
    L.check(lib.tq_init(0))
    return lib


def _nulls_on_edges(rng, n, p):
    """NOT-NULL bools with NULL runs across 64-row boundaries"""
    nn = rng.random(n) >= p
    for e in range(64, n, 192):
        nn[max(0, e - 3): e + 3] = False
    return nn


def _exact_cap(types, group_by, shards_host, W):
    """the most partial rows one source sends one destination (at least 1)"""
    most = 1
    for vals, nns in shards_host:
        n = len(vals[0]) if vals else 0
        if n == 0:
            continue
        if not group_by:
            continue
        want = RA.oracle(types, [(vals, nns)], group_by, [(FIRSTROW, g) for g in group_by])
        d = _dest_of(want.cols, types, group_by, W)
        most = max(most, int(np.bincount(d, minlength=W).max()))
    return most


def _dest_of(key_cols, types, group_by, W):
    n = key_cols[0].length
    return RA.group_dest(n, [np.ascontiguousarray(c.values).view(np.uint64) for c in key_cols], [c.not_null() for c in key_cols],
                         [types[g] == F64 for g in group_by], W)


def _check(lib, W, types, group_by, funcs, shards_host, loose=(), not_null=(), cap=None, reg=None, epoch=1):
    """run the exchange (funcs must end with FIRSTROW of every GROUP BY item) and compare; loose: result columns that only need
    to hold some value of their group (FIRSTROW of a non-key column).  Returns the per-rank results."""
    w = RA.width(lib, RA.desc(types, group_by, funcs)[0])
    cap = cap or _exact_cap(types, group_by, shards_host, W)
    own = reg is None
    reg = reg or X.Regions(lib, W, w + 1, cap)
    srcs = [R.Source(lib, [np.asarray(v).view(np.uint64) for v in vals], nns) for vals, nns in shards_host]
    try:
        out = RA.run(lib, W, types, group_by, funcs, srcs, reg, epoch, not_null)
    finally:
        for s in srcs:
            s.free()
        if own:
            reg.free()
    assert all(st == L.TQ_OK for st, _ in out), [st for st, _ in out]
    want = RA.oracle(types, shards_host, group_by, funcs)
    k = len(group_by)
    results = [cols for _, cols in out]
    if group_by:
        for q, cols in enumerate(results):
            if cols[0].length:
                d = _dest_of(cols[len(funcs) - k:], types, group_by, W)
                assert np.all(d == q), f"rank {q} finished groups another rank owns"
    else:
        assert all(c is None for c in results[1:]), "a scalar aggregate is finished on rank 0 only"
    from tinysql_b200.chunk import Chunk
    got = Chunk.concat([Chunk(c) for c in results if c is not None], [c.tp for c in want.cols]).cols
    assert got[0].length == want.cols[0].length, (got[0].length, want.cols[0].length)
    assert np.array_equal(RA.canon(got, loose), RA.canon(want.cols, loose)), "the groups differ from the oracle"
    if loose:
        _check_loose(got, funcs, loose, shards_host, types, group_by)
    return results


def _check_loose(got, funcs, loose, shards_host, types, group_by):
    """FIRSTROW of a non-key column: some value of its group"""
    k = len(group_by)
    keys_in = [np.concatenate([np.asarray(v[g]).view(np.uint64) for v, _ in shards_host]) for g in group_by]
    nn_in = [np.concatenate([nn[g] if nn[g] is not None else np.ones(len(v[g]), bool) for v, nn in shards_host]) for g in group_by]

    def norm(bits, nn, t):
        bits = np.where(nn, bits, np.uint64(0))
        return np.where((t == F64) & (bits == RA.NEG_ZERO), np.uint64(0), bits)
    key_rows = np.stack([norm(keys_in[i], nn_in[i], types[g]) for i, g in enumerate(group_by)] + [x.astype(np.uint64) for x in nn_in], 1)
    kc = got[len(funcs) - k:]
    got_keys = np.stack([norm(np.ascontiguousarray(c.values).view(np.uint64), c.not_null(), types[g]) for c, g in zip(kc, group_by)] +
                        [c.not_null().astype(np.uint64) for c in kc], 1)
    for i in loose:
        arg = funcs[i][1]
        col_in = np.concatenate([np.asarray(v[arg]).view(np.uint64) for v, _ in shards_host])
        nn_col = np.concatenate([nn[arg] if nn[arg] is not None else np.ones(len(v[arg]), bool) for v, nn in shards_host])
        gv, gn = np.ascontiguousarray(got[i].values).view(np.uint64), got[i].not_null()
        for r in range(got[i].length):
            rows = np.flatnonzero(np.all(key_rows == got_keys[r], axis=1))
            cand = set(zip(nn_col[rows].tolist(), np.where(nn_col[rows], col_in[rows], 0).tolist()))
            assert (bool(gn[r]), int(gv[r]) if gn[r] else 0) in cand, f"FIRSTROW column {i}, group {r}: not a value of its group"


def _dyadic(rng, n):
    return rng.integers(-4000, 4000, n) * 0.25


def _shards_types(rng, W, sizes, n_keys=300):
    """shards over (k INT64, x INT64, u UINT64, f DOUBLE): NULL keys, NULLs on 64-row edges, all-NULL groups (keys >= 290 have
    x and f NULL), u with the sign bit set"""
    out = []
    for r in range(W):
        n = sizes[r]
        k = rng.integers(0, n_keys, n).astype(np.int64)
        x = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
        u = rng.integers(0, 1 << 63, n, dtype=np.uint64) | (rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63))
        f = _dyadic(rng, n)
        knn = rng.random(n) >= 0.02
        xnn = _nulls_on_edges(rng, n, 0.1) & (k < 290)
        fnn = _nulls_on_edges(rng, n, 0.05) & (k < 290)
        out.append(([k, x, u, f], [knn, xnn, None, fnn]))
    return out


FUNCS_WIDE = [(COUNT, 1), (COUNT, -1), (SUM, 1), (AVG, 1), (MAX, 2), (MIN, 3), (SUM, 3), (AVG, 3), (MAX, 3), (FIRSTROW, 2), (FIRSTROW, 0)]


@pytest.mark.parametrize("W", WS)
def test_region_agg_functions_types_and_nulls(lib, W):
    """COUNT / COUNT(*) / SUM / AVG / MAX / MIN / FIRSTROW over INT64, UINT64 and DOUBLE with nullable arguments and NULL
    keys on several ranks: a 13-word partial row (+ the mask word); rank 1 brings an empty shard when W > 1"""
    rng = np.random.default_rng(W)
    sizes = [20_000 + 3_001 * r for r in range(W)]
    if W > 1:
        sizes[1] = 0
    _check(lib, W, [I64, I64, U64, F64], [0], FUNCS_WIDE, _shards_types(rng, W, sizes), loose=(9,))


@pytest.mark.parametrize("W", [2, 8])
def test_region_agg_rank_without_groups(lib, W):
    """every key names rank 0 (and no NULL key): the other ranks merge nothing and finish no group"""
    rng = np.random.default_rng(40 + W)
    keys = X.keys_to(rng, W, 0, 50)
    shards = []
    for r in range(W):
        k = rng.choice(keys, 5000)
        shards.append(([k, rng.integers(0, 100, 5000).astype(np.int64)], [None, None]))
    res = _check(lib, W, [I64, I64], [0], [(SUM, 1), (COUNT, -1), (FIRSTROW, 0)], shards, not_null=(0, 1))
    assert res[0][0].length == 50 and all(c[0].length == 0 for c in res[1:])


@pytest.mark.parametrize("W", WS)
def test_region_agg_multi_key(lib, W):
    """GROUP BY of 2 and 3 items mixing INT64, UINT64 (sign bit set) and DOUBLE, with NULL items and +0.0 / -0.0 on different
    ranks (the zero as the first and as the second item): each group made once"""
    rng = np.random.default_rng(100 + W)
    for layout in ([I64, F64], [U64, F64, I64], [F64, U64]):
        shards = []
        for r in range(W):
            n = 4000 + 500 * r
            cols, nns = [], []
            for g, t in enumerate(layout):
                if t == F64:
                    zero = -0.0 if r % 2 else 0.0
                    v = np.where(rng.random(n) < 0.5, zero, rng.integers(0, 4, n) * 0.5)
                elif t == U64:
                    v = rng.integers(0, 3, n).astype(np.uint64) | (rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63))
                else:
                    v = rng.integers(-3, 3, n).astype(np.int64)
                cols.append(v)
                nns.append(rng.random(n) >= 0.1)
            cols.append(_dyadic(rng, n))
            nns.append(rng.random(n) >= 0.2)
            shards.append((cols, nns))
        k = len(layout)
        types = layout + [F64]
        funcs = [(COUNT, -1), (SUM, k), (MAX, k)] + [(FIRSTROW, g) for g in range(k)]
        _check(lib, W, types, list(range(k)), funcs, shards)


@pytest.mark.parametrize("W", [1, 3])
def test_region_agg_scalar(lib, W):
    """no GROUP BY: every partial row goes to rank 0, which finishes the one row; with every shard empty it is COUNT 0 and
    NULL for the rest"""
    rng = np.random.default_rng(7)
    funcs = [(COUNT, -1), (COUNT, 1), (SUM, 1), (MAX, 0)]
    empty = [([np.zeros(0, np.int64), np.zeros(0, np.int64)], [None, None]) for _ in range(W)]
    res = _check(lib, W, [I64, I64], [], funcs, empty)
    assert res[0][0].length == 1 and res[0][0].values[0] == 0 and res[0][1].values[0] == 0
    assert not res[0][2].not_null()[0] and not res[0][3].not_null()[0]
    full = [([rng.integers(-99, 99, 1000).astype(np.int64), rng.integers(-99, 99, 1000).astype(np.int64)], [None, rng.random(1000) > 0.5])
            for _ in range(W)]
    _check(lib, W, [I64, I64], [], funcs, full)


def test_region_agg_cap_exact_and_one_short(lib):
    """a cap that fits the largest region exactly merges everything; one row short, the overflowing source publishes ~0 in
    every slot: every destination refuses with TQ_ERR_OOM and merges nothing"""
    W = 3
    rng = np.random.default_rng(11)
    shards = [([rng.integers(0, 5000, 8000).astype(np.int64), rng.integers(0, 9, 8000).astype(np.int64)], [None, None]) for _ in range(W)]
    types, funcs = [I64, I64], [(SUM, 1), (FIRSTROW, 0)]
    cap = _exact_cap(types, [0], shards, W)
    _check(lib, W, types, [0], funcs, shards, cap=cap)
    w = RA.width(lib, RA.desc(types, [0], funcs)[0])
    reg = X.Regions(lib, W, w + 1, cap - 1)
    srcs = [R.Source(lib, [np.asarray(v).view(np.uint64) for v in vals], nns) for vals, nns in shards]
    try:
        out = RA.run(lib, W, types, [0], funcs, srcs, reg)
        assert all(st == L.TQ_ERR_OOM for st, _ in out), [st for st, _ in out]
        for q in range(W):
            for g in range(W):
                rows, _ = reg.slots(q)[g]
                assert rows <= cap - 1 or rows == (1 << 64) - 1
                for c in range(w + 1):
                    assert np.all(reg.region(q, g, c)[cap - 1:] == X.SENTINEL), "a write past the cap"
    finally:
        for s in srcs:
            s.free()
        reg.free()


def test_region_agg_two_steps_reuse_regions(lib):
    """the second step pushes into the same regions under a new epoch and sees only its own rows"""
    W = 3
    rng = np.random.default_rng(12)
    types, funcs = [I64, I64], [(SUM, 1), (COUNT, -1), (FIRSTROW, 0)]
    w = RA.width(lib, RA.desc(types, [0], funcs)[0])
    reg = X.Regions(lib, W, w + 1, 4096)
    try:
        for epoch, n_keys in ((1, 3000), (2, 700)):
            shards = [([rng.integers(0, n_keys, 6000).astype(np.int64), rng.integers(0, 50, 6000).astype(np.int64)], [rng.random(6000) > 0.05, None])
                      for _ in range(W)]
            _check(lib, W, types, [0], funcs, shards, reg=reg, epoch=epoch)
    finally:
        reg.free()


def test_region_agg_refusals_write_nothing(lib):
    """a var-len GROUP BY, a FinalMode handle, a handle that merged partial rows, and bad arguments are refused before any
    region or slot is written; a merge into a handle fed raw rows, a FinalMode handle or with bad arguments too"""
    W = 2
    types, funcs = [I64, I64], [(SUM, 1), (FIRSTROW, 0)]
    d, keep = RA.desc(types, [0], funcs)
    w = RA.width(lib, d)
    reg = X.Regions(lib, W, w + 1, 64)
    src = R.Source(lib, [np.arange(100, dtype=np.uint64), np.arange(100, dtype=np.uint64)], [None, None])
    handles = []

    def untouched():
        ok = all(s == (0, 0) for q in range(W) for s in reg.slots(q))
        return ok and all(np.all(reg.region(q, g, c) == X.SENTINEL) for q in range(W) for g in range(W) for c in range(w + 1))
    try:
        h = RA.partial_handle(lib, d, src)
        handles.append(h)
        dest, cnts = reg.push_tables(0, 0)
        bad = [(0, dest, cnts, 64, 0), (9, dest, cnts, 64, 0), (W, None, cnts, 64, 0), (W, dest, None, 64, 0), (W, dest, cnts, 0, 0),
               (W, dest, cnts, 1 << 32, 0), (W, dest, cnts, 64, -1), (W, dest, cnts, 64, 16)]
        for n_parts, dd, cc, cap, slot in bad:
            assert lib.tq_agg_push_partial(h, n_parts, dd, cc, cap, slot, 1) == L.TQ_ERR_INVALID_ARG, (n_parts, cap, slot)
        holes = (C.c_void_p * len(dest))(*[dest[i] for i in range(len(dest))])
        holes[len(dest) - 1] = None
        assert lib.tq_agg_push_partial(h, W, holes, cnts, 64, 0, 1) == L.TQ_ERR_INVALID_ARG
        # var-len GROUP BY
        dv, kv = RA.desc([L.TQ_TYPE_BYTES, I64], [0], funcs)
        hv = RA.create(lib, dv)
        handles.append(hv)
        assert lib.tq_agg_push_partial(hv, W, dest, cnts, 64, 0, 1) == L.TQ_ERR_UNSUPPORTED_TYPE
        assert lib.tq_agg_merge_regions(hv, W, C.c_void_p(reg.slot_ptr(0, 0, 0)), 64, reg.region_table(0, 0)) == L.TQ_ERR_UNSUPPORTED_TYPE
        # FinalMode handle
        it = (C.c_int32 * 2)(I64, I64)
        gb = (C.c_int32 * 1)(0)
        ff = (L.TQAggFinalFunc * 1)(L.TQAggFinalFunc(SUM, 1, -1))
        fd = L.TQAggFinalDesc(2, it, 1, gb, 1, ff, 0)
        hf = C.c_void_p()
        L.check(lib.tq_agg_create_final(C.byref(fd), C.byref(hf)))
        handles.append(hf)
        assert lib.tq_agg_push_partial(hf, W, dest, cnts, 64, 0, 1) == L.TQ_ERR_STATE
        assert lib.tq_agg_merge_regions(hf, W, C.c_void_p(reg.slot_ptr(0, 0, 0)), 64, reg.region_table(0, 0)) == L.TQ_ERR_STATE
        # raw rows and partial rows on one handle
        assert lib.tq_agg_merge_regions(h, W, C.c_void_p(reg.slot_ptr(0, 0, 0)), 64, reg.region_table(0, 0)) == L.TQ_ERR_STATE
        hm = RA.create(lib, d)
        handles.append(hm)
        regs = reg.region_table(0, 0)
        for n_regions, slots, cap in ((0, reg.slot_ptr(0, 0, 0), 64), (9, reg.slot_ptr(0, 0, 0), 64), (W, None, 64), (W, reg.slot_ptr(0, 0, 0), 0)):
            assert lib.tq_agg_merge_regions(hm, n_regions, C.c_void_p(slots) if slots else None, cap, regs) == L.TQ_ERR_INVALID_ARG
        regs[1].data = None
        assert lib.tq_agg_merge_regions(hm, W, C.c_void_p(reg.slot_ptr(0, 0, 0)), 64, regs) == L.TQ_ERR_INVALID_ARG
        X.compute_sync(lib)
        assert untouched(), "a refused call wrote a region or a slot"
        # a handle that merged partial rows cannot push
        regs = reg.region_table(0, 0)
        assert lib.tq_agg_merge_regions(hm, W, C.c_void_p(reg.slot_ptr(0, 0, 0)), 64, regs) == L.TQ_OK   # all slots read 0 rows
        assert lib.tq_agg_push_partial(hm, W, dest, cnts, 64, 0, 1) == L.TQ_ERR_STATE
        X.compute_sync(lib)
        assert untouched()
    finally:
        for hh in handles:
            lib.tq_agg_destroy(hh)
        src.free()
        reg.free()
