"""GPU suite: ORDER BY and ORDER BY ... LIMIT across ranks (tq_partition_push_sample -> tq_partition_push_ranges ->
tq_sort_put_regions) through dist.RegionSort, with W ranks emulated in one process (tests/region_sort_ref.py).  The ranks'
outputs concatenated in rank order must equal, row for row and payload included, the single-GPU tq_sort of the shards
concatenated in rank order, and sort_ref.sort_rows of the same rows."""
import ctypes as C

import numpy as np
import pytest

import region_sort_ref as RS
import sort_ref as SR
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, Column, VarColumn

pytestmark = pytest.mark.gpu

I64, U64, F64, F32 = L.TQ_TYPE_INT64, L.TQ_TYPE_UINT64, L.TQ_TYPE_FLOAT64, L.TQ_TYPE_FLOAT32
WS = [1, 2, 3, 8]


@pytest.fixture(scope="module")
def lib():
    lib = L.load()
    L.check(lib.tq_init(0))
    return lib


def _col(tp, vals):
    return SR.column(tp, vals, nullable=any(v is None for v in vals))


def _gen(rng, tp, n, p_null=0.1, distinct=None):
    pools = {I64: [SR.INT64_MIN, -1, 0, 1, SR.INT64_MAX], U64: [0, 1, 1 << 63, SR.UINT64_MAX], F64: [-0.0, 0.0, -1.5, float("inf")],
             BYTES: [b"", b"\0", b"abcdefgh", b"abcdefgh\0", b"abcdefghijklmnop", b"abcdefghijklmnopq"]}
    out = []
    for _ in range(n):
        if rng.random() < p_null:
            out.append(None)
        elif rng.random() < 0.3:
            out.append(pools[tp][int(rng.integers(0, len(pools[tp])))])
        elif tp == I64:
            out.append(int(rng.integers(-(distinct or 1 << 62), distinct or 1 << 62)))
        elif tp == U64:
            out.append(int(rng.integers(0, distinct or 1 << 63)) | (int(rng.integers(0, 2)) << 63 if distinct is None else 0))
        elif tp == F64:
            out.append(float(rng.integers(-(distinct or 1000), distinct or 1000)) / 4)
        else:
            out.append(rng.integers(97, 100 if distinct else 123, int(rng.integers(0, 20))).astype(np.uint8).tobytes())
    return out


def single_sort(lib, types, cols, by, offset=0, count=-1):
    """the one-GPU tq_sort of host Columns: rows of Python values"""
    n = cols[0].length
    tt = (C.c_int32 * len(types))(*types)
    bc = (C.c_int32 * max(len(by), 1))(*[c for c, _ in by])
    bd = (C.c_int32 * max(len(by), 1))(*[int(d) for _, d in by])
    d = L.TQSortDesc(len(types), tt, len(by), bc, bd, offset, count)
    h = C.c_void_p()
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    try:
        if n:
            L.check(lib.tq_sort_put(h, (L.TQColumn * len(cols))(*[c.tq() for c in cols]), L.TQ_MEM_HOST))
        L.check(lib.tq_sort_eof(h))
        nb = max([int(c.offsets[-1]) for c in cols if c.tp == BYTES] + [1])
        outs = [VarColumn.empty(t, max(n, 1), nb) if t == BYTES else Column.empty(t, max(n, 1)) for t in types]
        rows, eof = C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_sort_next(h, max(n, 1), (L.TQColumn * len(types))(*[o.tq() for o in outs]), C.byref(rows), C.byref(eof)))
        k = rows.value
        res = [o.head(k) if t == BYTES else Column(t, o.values[:k], o.not_null()[:k]) for o, t in zip(outs, types)]
        return RS.rows_of(res) if k else []
    finally:
        lib.tq_sort_destroy(h)


def _byte_caps(types, shards):
    return [max([int(sh[c].offsets[-1]) for sh in shards] + [1]) if t == BYTES else None for c, t in enumerate(types)]


def _check(lib, W, types, by, shards, offset=0, count=-1, n_samples=1024, em=None):
    """one step on W emulated ranks: the rank-major concatenation of the outputs == one-GPU tq_sort == sort_ref; TopN only on
    rank 0.  Returns the rows per rank"""
    n_max = max(sh[0].length for sh in shards)
    own = em is None
    em = em or RS.Emulated(lib, W, types, [c for c, _ in by], [d for _, d in by], n_max, _byte_caps(types, shards), True, offset, count,
                           n_samples)
    try:
        out = em.step(shards)
    finally:
        if own:
            em.free()
    allcols = RS.concat(shards, types)
    got = [r for rows, res in out if res is not None for r in RS.rows_of(res)]
    assert [rows for rows, _ in out] == [0 if res is None else res[0].length for _, res in out]
    want = SR.sort_rows(RS.rows_of(allcols), by, offset, count)
    assert SR.canon_rows(got) == SR.canon_rows(want), "the ranks' outputs differ from sort_ref"
    assert SR.canon_rows(got) == SR.canon_rows(single_sort(lib, types, allcols, by, offset, count)), "differs from the one-GPU tq_sort"
    if count >= 0:
        assert all(rows == 0 for rows, _ in out[1:]), "TopN rows on a rank other than 0"
    return [rows for rows, _ in out]


@pytest.mark.parametrize("W", WS)
def test_every_type_as_key_and_payload(lib, W):
    """INT64 / UINT64 / FLOAT64 / BYTES each as key (ASC and DESC mixed, NULLs) with the others as payload"""
    rng = np.random.default_rng(W)
    types = [I64, U64, F64, BYTES]
    shards = [[_col(t, _gen(rng, t, 700 + 97 * r)) for t in types] for r in range(W)]
    for by in ([(0, False)], [(1, True)], [(2, False), (0, True)], [(3, True), (2, False)], [(3, False), (1, False), (2, True), (0, False)]):
        _check(lib, W, types, by, shards)


@pytest.mark.parametrize("W", WS)
def test_sorted_reverse_and_duplicate_inputs(lib, W):
    """already sorted, reverse sorted and all-duplicate keys: exact, and an all-duplicate column spreads over the ranks"""
    n = 3000
    base = np.arange(W * n, dtype=np.int64)
    for keys in (base, base[::-1].copy(), np.full(W * n, 42, np.int64)):
        pay = np.arange(W * n, dtype=np.int64) * 7
        shards = [[Column(I64, keys[r * n:(r + 1) * n]), Column(I64, pay[r * n:(r + 1) * n])] for r in range(W)]
        rows = _check(lib, W, [I64, I64], [(0, False)], shards)
        if W > 1:
            assert max(rows) < W * n, f"one rank received every row: {rows}"


@pytest.mark.parametrize("W", [2, 3, 8])
def test_empty_shards(lib, W):
    """some shards empty, then every shard empty"""
    rng = np.random.default_rng(50 + W)
    types = [BYTES, I64]
    for sizes in ([0] + [500] * (W - 1), [500] + [0] * (W - 1), [0] * W):
        shards = [[_col(BYTES, _gen(rng, BYTES, k)), _col(I64, _gen(rng, I64, k))] for k in sizes]
        _check(lib, W, types, [(0, True), (1, False)], shards)


@pytest.mark.parametrize("W", WS)
def test_topn_windows(lib, W):
    """TopN windows that span ranks, limit_count 0 and a window past the total, on rank 0"""
    rng = np.random.default_rng(70 + W)
    types = [F64, BYTES, I64]
    shards = [[_col(t, _gen(rng, t, 400 + 13 * r, distinct=50)) for t in types] for r in range(W)]
    total = sum(sh[0].length for sh in shards)
    for offset, count in ((0, 10), (350, 500), (0, 0), (total - 5, 100), (total + 10, 5), (0, total + 1)):
        _check(lib, W, types, [(0, True), (1, False)], shards, offset, count)


def test_two_steps_reuse_regions(lib):
    """the second step pushes into the same regions under a new epoch and sees only its own rows"""
    W = 3
    rng = np.random.default_rng(90)
    types = [I64, BYTES]
    em = RS.Emulated(lib, W, types, [1, 0], [False, True], 2000, [60_000, 60_000], True)
    try:
        for n in (2000, 300):
            shards = [[_col(I64, _gen(rng, I64, n)), _col(BYTES, _gen(rng, BYTES, n))] for _ in range(W)]
            _check(lib, W, types, [(1, False), (0, True)], shards, em=em)
    finally:
        em.free()


def test_byte_cap_overflow_fails_every_rank(lib):
    """a destination's cells past the byte cap: every rank's step fails and no rank returns a result"""
    W = 3
    n = 1000
    types = [BYTES]
    shards = [[VarColumn(BYTES, [b"%010d" % (r * n + i) for i in range(n)])] for r in range(W)]
    em = RS.Emulated(lib, W, types, [0], [False], n, [n * 10 // 2], False, n_samples=64)
    failed = []
    try:
        em.ex.next_epoch()
        dev = [RS.device(sh) for sh in shards]
        try:
            for r in range(W):
                em.sorts[r].push_sample(dev[r])
            for r in range(W):
                em.sorts[r].push_rows(dev[r])
            for r in range(W):
                with pytest.raises(L.TQError) as ei:
                    em.sorts[r].finish(keep_result=True)
                failed.append(ei.value.status)
        finally:
            for s in em.sorts:
                s.release()
            for d in dev:
                for c in d:
                    c.free()
    finally:
        em.free()
    assert failed == [L.TQ_ERR_OOM] * W


def test_refusals_write_nothing(lib):
    """FLOAT32, bad n_parts, decreasing splitter positions and a null destination are refused before anything is enqueued:
    no region and no slot changes"""
    W = 3
    types = [I64, BYTES]
    em = RS.Emulated(lib, W, types, [0], [False], 64, [1024, 1024], True)
    sh = [Column(I64, np.arange(10, dtype=np.int64)), VarColumn(BYTES, [b"x"] * 10)]
    dev = RS.device(sh)
    try:
        arr = (L.TQColumn * 2)(*[c.tq() for c in dev])
        before = em.ex.buf.get(np.uint8)
        by, desc = (C.c_int32 * 1)(0), (C.c_int32 * 1)(0)
        caps = (C.c_int64 * 2)(0, 1024)
        dest, cnts = em.ex.push_tables(1, 0)
        sdest, scnts = em.ex.push_tables(0, 0)
        spl = (L.TQColumn * 2)(*[c.tq() for c in dev])

        def ranges(tt, n_parts, pos, d=dest):
            return lib.tq_partition_push_ranges(2, arr, (C.c_int32 * 2)(*tt), 10, 1, by, desc, 0, n_parts, spl, 10, (C.c_int64 * max(len(pos), 1))(*pos),
                                                d, cnts, em.ex.cap[1], caps, 0, 1)
        assert ranges([F32, BYTES], 3, [3, 4]) == L.TQ_ERR_UNSUPPORTED_TYPE
        assert ranges([I64, BYTES], 0, []) == L.TQ_ERR_INVALID_ARG
        assert ranges([I64, BYTES], 9, [0] * 8) == L.TQ_ERR_INVALID_ARG
        assert ranges([I64, BYTES], 3, [5, 2]) == L.TQ_ERR_INVALID_ARG          # splitter positions decrease
        assert ranges([I64, BYTES], 3, [5, 10]) == L.TQ_ERR_INVALID_ARG         # past the splitter rows
        nulld = (C.c_void_p * len(dest))(*dest)
        nulld[4] = None
        assert ranges([I64, BYTES], 3, [3, 4], nulld) == L.TQ_ERR_INVALID_ARG
        assert lib.tq_partition_push_sample(2, arr, (C.c_int32 * 2)(F32, BYTES), 10, 1, by, 1, 0, 16, 7, W, sdest, scnts, em.ex.cap[0], caps, 0,
                                            1) == L.TQ_ERR_UNSUPPORTED_TYPE
        assert lib.tq_partition_push_sample(2, arr, (C.c_int32 * 2)(I64, BYTES), 10, 1, by, 1, 0, 0, 7, W, sdest, scnts, em.ex.cap[0], caps, 0,
                                            1) == L.TQ_ERR_INVALID_ARG
        L.check(lib.tq_partition_push_sync(0))
        assert np.array_equal(em.ex.buf.get(np.uint8), before), "a refused push wrote a region or a slot"
    finally:
        for c in dev:
            c.free()
        em.free()
