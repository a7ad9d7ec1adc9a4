"""GPU suite: GROUP BY over string columns across ranks (tq_agg_push_partial_var -> tq_region_wait ->
tq_agg_merge_regions_var) through dist.RegionAgg, with W ranks emulated in one process (tests/region_agg_strings_ref.py).
The union of the ranks' results must equal oracle_py.hash_agg over every shard, every group must be finished on the rank
the destination twin names, and FIRSTROW of a non-key column must hold a value of its group."""
import ctypes as C

import numpy as np
import pytest

import exchange_ref as X
import region_agg_ref as RA
import region_agg_strings_ref as S
import region_outer_ref as R
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, Column, VarColumn
from tinysql_b200.dist import RegionAgg, partial_var_cols

pytestmark = pytest.mark.gpu

COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)
I64, F64 = L.TQ_TYPE_INT64, L.TQ_TYPE_FLOAT64
WS = [1, 2, 3, 8]


@pytest.fixture(scope="module")
def lib():
    lib = L.load()
    L.check(lib.tq_init(0))
    return lib


def _words(rng, k, lo=0, hi=24):
    """k distinct strings of lo..hi bytes, "" among them"""
    out = {b""}
    while len(out) < k:
        out.add(rng.integers(97, 123, int(rng.integers(max(lo, 1), hi + 1)), dtype=np.uint8).tobytes())
    return sorted(out)


def _scol(rng, words, n, p_null):
    vals = [words[i] for i in rng.integers(0, len(words), n)]
    return VarColumn(BYTES, [None if rng.random() < p_null else v for v in vals])


def _check(lib, W, types, group_by, funcs, shards, loose=(), max_groups=None, em=None):
    """run one step and compare with the oracle (funcs end with FIRSTROW of every GROUP BY item); loose: result columns that
    only need some value of their group (FIRSTROW of a non-key column)"""
    caps = S.byte_caps(types, group_by, funcs, shards)
    own = em is None
    em = em or S.Emulated(lib, W, types, group_by, funcs, max_groups or max(sh[0].length for sh in shards) + 1, caps)
    try:
        results = em.step(shards)
    finally:
        if own:
            em.free()
    want = S.oracle(types, shards, group_by, funcs)
    k = len(group_by)
    got_rows = []
    for q, res in enumerate(results):
        if res is None:
            continue
        if res[0].length and group_by:
            assert np.all(S.dest_of(res[len(funcs) - k:], types, group_by, W) == q), f"rank {q} finished groups another rank owns"
        got_rows += S.rows_of(res, loose)
    if not group_by:
        assert all(r is None for r in results[1:]), "a scalar aggregate is finished on rank 0 only"
    assert sorted(got_rows, key=lambda r: tuple((x is None, repr(x)) for x in r)) == S.rows_of(want, loose), "the groups differ from the oracle"
    if loose:
        full = S.concat(shards, types)
        for i in loose:
            arg = funcs[i][1]
            member = {}
            for key, v in zip(zip(*[full[g].tolist() if full[g].tp == BYTES else _plain(full[g]) for g in group_by]),
                              full[arg].tolist() if full[arg].tp == BYTES else _plain(full[arg])):
                member.setdefault(key, set()).add(v)
            for res in results:
                if res is None:
                    continue
                kc = res[len(funcs) - k:]
                for key, v in zip(zip(*[c.tolist() if c.tp == BYTES else _plain(c) for c in kc]), res[i].tolist() if res[i].tp == BYTES else _plain(res[i])):
                    assert v in member[key], f"FIRSTROW column {i}: {v!r} is not a value of group {key!r}"
    return results


def _plain(c):
    return [None if not ok else (float(v) + 0.0 if c.tp == F64 else int(v)) for v, ok in zip(c.values, c.not_null())]


@pytest.mark.parametrize("W", WS)
def test_string_group_by_with_string_max_min(lib, W):
    """GROUP BY s alone, with MAX(s) / MIN(s) / COUNT(s) on the same column, MAX / MIN / FIRSTROW of another string column t
    and SUM(x): NULL and "" are different groups; rank 1 brings an empty shard when W > 1"""
    rng = np.random.default_rng(W)
    words, other = _words(rng, 400), _words(rng, 300, 0, 300)
    shards = []
    for r in range(W):
        n = 0 if (W > 1 and r == 1) else 6000 + 700 * r
        shards.append([_scol(rng, words, n, 0.05), _scol(rng, other, n, 0.2), Column(I64, rng.integers(-1000, 1000, n).astype(np.int64),
                                                                                       rng.random(n) >= 0.1)])
    types = [BYTES, BYTES, I64]
    funcs = [(COUNT, -1), (SUM, 2), (MAX, 0), (MIN, 0), (COUNT, 0), (MAX, 1), (MIN, 1), (COUNT, 1), (FIRSTROW, 1), (FIRSTROW, 0)]
    _check(lib, W, types, [0], funcs, shards, loose=(8,))


@pytest.mark.parametrize("W", WS)
def test_string_multi_item_keys(lib, W):
    """GROUP BY (s, k INT64, f DOUBLE) with NULL items and both zeros, and (k, s): each group made once, on its rank"""
    rng = np.random.default_rng(20 + W)
    words = _words(rng, 30)
    shards = []
    for r in range(W):
        n = 4000 + 300 * r
        f = np.where(rng.random(n) < 0.4, -0.0 if r % 2 else 0.0, rng.integers(0, 3, n) * 0.5)
        shards.append([_scol(rng, words, n, 0.1), Column(I64, rng.integers(-3, 3, n).astype(np.int64), rng.random(n) >= 0.1),
                       Column(F64, f, rng.random(n) >= 0.1), Column(F64, rng.integers(-400, 400, n) * 0.25, rng.random(n) >= 0.2)])
    types = [BYTES, I64, F64, F64]
    _check(lib, W, types, [0, 1, 2], [(COUNT, -1), (SUM, 3), (MAX, 0), (FIRSTROW, 0), (FIRSTROW, 1), (FIRSTROW, 2)], shards)
    _check(lib, W, types, [1, 0], [(AVG, 3), (MIN, 0), (FIRSTROW, 1), (FIRSTROW, 0)], shards)


@pytest.mark.parametrize("W", [2, 8])
def test_string_group_by_high_ndv(lib, W):
    """100k distinct strings of 1..64 bytes over 200k rows: most groups have one row on one rank"""
    rng = np.random.default_rng(30 + W)
    words = _words(rng, 100_000, 1, 64)
    n = 200_000 // W
    shards = [[_scol(rng, words, n, 0.01), Column(I64, rng.integers(0, 9, n).astype(np.int64))] for _ in range(W)]
    _check(lib, W, [BYTES, I64], [0], [(SUM, 1), (COUNT, -1), (FIRSTROW, 0)], shards)


def test_string_two_steps_reuse_regions(lib):
    """the second step pushes into the same regions under a new epoch and sees only its own rows"""
    W = 3
    rng = np.random.default_rng(40)
    types, funcs = [BYTES, I64], [(SUM, 1), (MAX, 0), (FIRSTROW, 0)]
    caps = [200_000, None]
    em = S.Emulated(lib, W, types, [0], funcs, 8000, caps)
    try:
        for k in (3000, 500):
            words = _words(rng, k)
            shards = [[_scol(rng, words, 6000, 0.05), Column(I64, rng.integers(0, 50, 6000).astype(np.int64))] for _ in range(W)]
            _check(lib, W, types, [0], funcs, shards, em=em)
    finally:
        em.free()


def test_string_byte_overflow_is_oom(lib):
    """cells past a region's byte area: the push publishes ~0, the merge is TQ_ERR_OOM and RegionLayout.counts raises"""
    W = 2
    rng = np.random.default_rng(50)
    words = _words(rng, 3000, 60, 100)
    types, funcs = [BYTES, I64], [(SUM, 1), (FIRSTROW, 0)]
    shards = [[VarColumn(BYTES, words), Column(I64, np.arange(len(words), dtype=np.int64))] for _ in range(W)]
    em = S.Emulated(lib, W, types, [0], funcs, 4000, [1, None])        # a byte area of 16 KiB: ~120 KB of cells per region
    try:
        with pytest.raises(L.TQError) as e:
            em.step(shards)
        assert e.value.status == L.TQ_ERR_OOM
        for q in range(W):
            with pytest.raises(RuntimeError):
                em.ex.counts(q)
    finally:
        em.free()


def _fixed_shards(rng, W):
    return [([rng.integers(0, 3000, 5000).astype(np.int64), rng.integers(-99, 99, 5000).astype(np.int64)], [rng.random(5000) > 0.05, None])
            for _ in range(W)]


def test_new_pair_equals_old_pair_on_fixed_width(lib):
    """on a handle without string columns tq_agg_push_partial_var publishes the slots tq_agg_push_partial publishes and
    writes the same rows into the same regions, and tq_agg_merge_regions_var finishes the same groups"""
    W = 3
    rng = np.random.default_rng(60)
    types, funcs = [I64, I64], [(SUM, 1), (COUNT, -1), (MAX, 1), (FIRSTROW, 0)]
    d, keep = RA.desc(types, [0], funcs)
    w = RA.width(lib, d)
    shards = _fixed_shards(rng, W)
    regs = [X.Regions(lib, W, w + 1, 4096) for _ in range(2)]
    srcs = [R.Source(lib, [np.asarray(v).view(np.uint64) for v in vals], nns) for vals, nns in shards]
    hs = []
    try:
        for new, reg in enumerate(regs):
            for s in range(W):
                hs.append(RA.partial_handle(lib, d, srcs[s]))
                dest, cnts = reg.push_tables(0, s)
                if new:
                    L.check(lib.tq_agg_push_partial_var(hs[-1], W, dest, cnts, 4096, None, s, 1))
                else:
                    L.check(lib.tq_agg_push_partial(hs[-1], W, dest, cnts, 4096, s, 1))
            for s in range(W):
                L.check(lib.tq_partition_push_sync(s))
        for q in range(W):
            assert regs[0].slots(q) == regs[1].slots(q)
            for g in range(W):
                # a handle exports its partial rows in table order, which differs between handles: compare each region's rows as
                # a multiset, and the words past them (the sentinel) as they are
                rows = regs[0].slots(q)[g][0]
                areas = [np.stack([r.region(q, g, c) for c in range(w + 1)], 1) for r in regs]
                assert np.array_equal(X.sorted_rows(areas[0][:rows]), X.sorted_rows(areas[1][:rows])), (q, g)
                assert np.array_equal(areas[0][rows:], areas[1][rows:]), (q, g)
            outs = []
            for merge in (lib.tq_agg_merge_regions, lib.tq_agg_merge_regions_var):
                L.check(regs[0].wait(q, 1))
                hf = RA.create(lib, d)
                try:
                    L.check(merge(hf, W, C.c_void_p(regs[0].slot_ptr(q, 0, 0)), 4096, regs[0].region_table(q, 0)))
                    L.check(lib.tq_agg_eof(hf))
                    outs.append(RA.canon(RA.agg_drain(lib, L, hf, len(funcs))))
                finally:
                    lib.tq_agg_destroy(hf)
            assert np.array_equal(outs[0], outs[1])
    finally:
        for h in hs:
            lib.tq_agg_destroy(h)
        for s in srcs:
            s.free()
        for reg in regs:
            reg.free()


def test_string_refusals_write_nothing(lib):
    """bad byte caps, a missing byte area, a string column without offsets on the merge, a FinalMode handle, and a string
    handle on the old pair are refused before any region or slot is written"""
    W = 2
    types, funcs = [BYTES, I64], [(SUM, 1), (MAX, 0), (FIRSTROW, 0)]
    var = partial_var_cols(types, [0], funcs)
    assert [c for c, _ in var] == [0, 2, 3]
    w = RA.width(lib, RA.desc(types, [0], funcs)[0])
    _, bcaps = RegionAgg.table_of(W, w, var, True, 64, [100, None])
    em = S.Emulated(lib, W, types, [0], funcs, 64, [100, None])
    ex = em.ex
    rng = np.random.default_rng(70)
    words = _words(rng, 50)
    shard = [_scol(rng, words, 100, 0.1), Column(I64, np.arange(100, dtype=np.int64))]
    dcols = S.device(shard)
    d, keep = RA.desc(types, [0], funcs)
    h = RA.create(lib, d)
    hm = RA.create(lib, d)

    def untouched():
        slots = ex.read_slots(0)[0].tolist() + ex.read_slots(1)[0].tolist()
        if any(s != [0, 0] for s in slots):
            return False
        raw = np.zeros(ex.bytes * W, np.uint8)
        L.check(lib.tq_memcpy_d2h(raw.ctypes.data, C.c_void_p(ex.bases[0]), raw.nbytes))
        return all(np.all(raw[b - ex.bases[0] + ex.reg_off[0]: b - ex.bases[0] + ex.bytes] == X.SENTINEL_BYTE) for b in ex.bases)
    try:
        from tinysql_b200.dist import _tq_device
        arr, n = _tq_device(L, dcols)
        L.check(lib.tq_agg_put(h, arr, L.TQ_MEM_DEVICE))
        L.check(lib.tq_agg_eof(h))
        dest, cnts = ex.push_tables(0, 0)
        cap = ex.cap[0]
        for bad in ([0, 8, 8], [-1, 8, 8], [8, 8, 1 << 32], [8, 0, 8]):
            bc = (C.c_int64 * 3)(*bad)
            assert lib.tq_agg_push_partial_var(h, W, dest, cnts, cap, bc, 0, 1) == L.TQ_ERR_INVALID_ARG, bad
        good = (C.c_int64 * 3)(*bcaps)
        assert lib.tq_agg_push_partial_var(h, W, dest, cnts, cap, None, 0, 1) == L.TQ_ERR_INVALID_ARG
        holes = (C.c_void_p * len(dest))(*[dest[i] for i in range(len(dest))])
        holes[len(dest) - 1] = None                      # the last byte area of the last destination
        assert lib.tq_agg_push_partial_var(h, W, holes, cnts, cap, good, 0, 1) == L.TQ_ERR_INVALID_ARG
        assert lib.tq_agg_push_partial_var(h, W, dest, cnts, 0, good, 0, 1) == L.TQ_ERR_INVALID_ARG
        assert lib.tq_agg_push_partial(h, W, dest, cnts, cap, 0, 1) == L.TQ_ERR_UNSUPPORTED_TYPE
        regs = em.aggs[0].merge_table(0)
        assert lib.tq_agg_merge_regions(hm, W, C.c_void_p(ex.slot_ptr(0, 0, 0)), cap, regs) == L.TQ_ERR_UNSUPPORTED_TYPE
        regs[w + 1].offsets = None                       # region 1's GROUP BY column
        assert lib.tq_agg_merge_regions_var(hm, W, C.c_void_p(ex.slot_ptr(0, 0, 0)), cap, regs) == L.TQ_ERR_INVALID_ARG
        it = (C.c_int32 * 2)(BYTES, I64)
        gb = (C.c_int32 * 1)(0)
        ff = (L.TQAggFinalFunc * 1)(L.TQAggFinalFunc(SUM, 1, -1))
        fd = L.TQAggFinalDesc(2, it, 1, gb, 1, ff, 0)
        hf = C.c_void_p()
        L.check(lib.tq_agg_create_final(C.byref(fd), C.byref(hf)))
        try:
            assert lib.tq_agg_push_partial_var(hf, W, dest, cnts, cap, good, 0, 1) == L.TQ_ERR_STATE
            assert lib.tq_agg_merge_regions_var(hf, W, C.c_void_p(ex.slot_ptr(0, 0, 0)), cap, em.aggs[0].merge_table(0)) == L.TQ_ERR_STATE
        finally:
            lib.tq_agg_destroy(hf)
        X.compute_sync(lib)
        assert untouched(), "a refused call wrote a region or a slot"
        # the same handle pushes once its arguments are right
        L.check(lib.tq_agg_push_partial_var(h, W, dest, cnts, cap, good, 0, 1))
        L.check(lib.tq_partition_push_sync(0))
        assert not untouched()
    finally:
        lib.tq_agg_destroy(h)
        lib.tq_agg_destroy(hm)
        for c in dcols:
            c.free()
        em.free()
