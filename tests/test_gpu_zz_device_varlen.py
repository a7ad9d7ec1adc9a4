"""GPU parity for var-len (string) columns that arrive in device memory (TQ_MEM_DEVICE puts): the hash join (keys and payloads,
build and probe), the hash aggregation (GROUP BY items, COUNT / MAX / MIN / FIRSTROW arguments, FinalMode partial columns),
sort / TopN ByItems and merge-join keys, and the chains that hand lent string columns from one operator to the next without
visiting the host.  Every result is checked against the oracle.  Cells cover NULL, empty, 1-7 bytes, exactly 8, more than 8
and more than 64 bytes; device columns are laid out with offsets[0] != 0 (a cell range inside a larger buffer).  The sort /
TopN / merge-join bodies also run under the CPU emulation (test_emu_device_varlen.py).  (The file name keeps these tests
last, with the other device-chain tests.)"""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import (BYTES, FLOAT32, INT64, Chunk, Column, DeviceChunk, DeviceColumn, DeviceVarColumn, VarColumn, device_to_host,
                                device_var_to_host, encode_chunk, pack_not_null, tq_array)
from tinysql_b200.executor import AGG_COUNT, AGG_FIRSTROW, AGG_MAX, AGG_MIN, AGG_SUM, INNER_JOIN, LEFT_OUTER_JOIN, RIGHT_OUTER_JOIN
from util import assert_same_multiset, assert_same_ordered

pytestmark = pytest.mark.gpu

LEADS = (0, 5, 8, 13)   # offsets[0] of the successive device pieces


LENS = (0, 1, 3, 7, 8, 9, 15, 16, 33, 64, 65, 100)


def cell_of(rng, v):
    """a string of one of the interesting lengths, a function of v: distinct for distinct v below 2^24, except that the
    lengths 0 and 1 only occur for v < 64 (so a join on these strings keeps a bounded result)"""
    ln = LENS[v % 12] if v < 64 else LENS[2 + v % 10]
    return ((v + 1).to_bytes(4, "little") * 26)[:ln]


def vocab(rng, n_words, null_frac, n, max_extra=0):
    """n cells drawn from n_words distinct strings (+ NULLs); max_extra > 0 adds that many random bytes to some cells"""
    words = [cell_of(rng, v) for v in range(n_words)]
    idx = rng.integers(0, n_words, n)
    nn = rng.random(n) >= null_frac
    out = [words[i] if ok else None for i, ok in zip(idx, nn)]
    if max_extra:
        for i in np.nonzero(rng.random(n) < 0.05)[0]:
            if out[i] is not None:
                out[i] = out[i] + bytes(rng.integers(0, 256, int(rng.integers(0, max_extra + 1)), dtype=np.uint8))
    return out


def piece(col, lo, hi):
    """rows [lo, hi) of a column (a var-len column is cut from its offsets / bytes without visiting the cells)"""
    if col.tp != BYTES:
        return col.slice(lo, hi)
    c = object.__new__(VarColumn)
    c.tp, c.length = BYTES, hi - lo
    c.offsets = col.offsets[lo: hi + 1] - col.offsets[lo]
    c.data = col.data[col.offsets[lo]: col.offsets[hi]]
    c.bitmap = None if col.bitmap is None else pack_not_null(col.not_null()[lo:hi])
    return c


def to_device(col, lead):
    return DeviceVarColumn.from_host(col, lead) if col.tp == BYTES else DeviceColumn.from_host(col)


def device_pieces(cols, bounds):
    """yield (device columns, tq_column array) for the row ranges [bounds[i], bounds[i + 1])"""
    for i in range(len(bounds) - 1):
        lo, hi = bounds[i], bounds[i + 1]
        dcs = [to_device(piece(c, lo, hi), LEADS[i % len(LEADS)]) for c in cols]
        yield dcs, (L.TQColumn * len(dcs))(*[d.tq() for d in dcs])


def scribble_cells(lib, dcs):
    """overwrite the offsets and bytes of every var-len device column (the call that took them must have copied them)"""
    for d in dcs:
        if isinstance(d, DeviceVarColumn):
            L.check(lib.tq_memset_device(d._off, 0xAB, d.off_bytes))
            L.check(lib.tq_memset_device(d._data, 0xCD, d.data_bytes))


def free_all(dcs):
    for d in dcs:
        d.free()


def column_to_host(tp, t, n):
    if tp == BYTES:
        return device_var_to_host(t.data, t.offsets, t.null_bitmap, n) if n else Column(BYTES, [])
    return device_to_host(tp, t.data, t.null_bitmap, n)


def lent_to_host(types, out, n):
    return Chunk([column_to_host(tp, out[i], n) for i, tp in enumerate(types)])


def i32(vals):
    return (C.c_int32 * max(len(vals), 1))(*vals)


# ------------------------------------------------------------------------------------------------------------- hash join
def join_device(lib, jt, oir, btypes, b, ptypes, p, bkeys, pkeys, bbounds, pbounds, batch=0):
    d = L.TQJoinDesc(jt, 1 if oir else 0, len(btypes), i32(btypes), len(ptypes), i32(ptypes), len(bkeys), i32(bkeys), i32(pkeys), batch, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    held = []
    for dcs, arr in device_pieces(b, bbounds):
        L.check(lib.tq_join_put_build(h, arr, L.TQ_MEM_DEVICE))
        scribble_cells(lib, dcs)     # var-len cells are copied by the put; 8-byte columns and bitmaps stay borrowed
        held.append(dcs)
    L.check(lib.tq_join_finalize_build(h))
    for dcs in held:
        free_all(dcs)
    otypes = (btypes + ptypes) if oir else (ptypes + btypes)
    out = (L.TQColumn * len(otypes))()
    n, eof = C.c_int64(0), C.c_int32(0)
    parts, prev = [], None

    def drain():
        while True:
            L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
            if n.value == 0:
                return
            parts.append(lent_to_host(otypes, out, n.value))

    for dcs, arr in device_pieces(p, pbounds):
        L.check(lib.tq_join_put_probe(h, arr, None, L.TQ_MEM_DEVICE))
        scribble_cells(lib, dcs)
        if prev is not None:
            free_all(prev)           # the batch that read it has been finalised by this put
        prev = dcs
        drain()
    L.check(lib.tq_join_probe_eof(h))
    if prev is not None:
        free_all(prev)
    drain()
    assert eof.value == 1
    L.check(lib.tq_join_destroy(h))
    return Chunk.concat(parts, otypes) if parts else Chunk([Column(BYTES, []) if t == BYTES else Column(t, np.zeros(0, np.int64)) for t in otypes])


def ragged_bounds(rng, n, mean, mult=8):
    """piece boundaries of varying size, multiples of `mult` except the last (device build chunks with NULL bitmaps
    must start at multiples of 8 rows)"""
    b, x = [0], 0
    while x < n:
        x = min(n, x + max(mult, int(rng.integers(mean // 2, mean * 3 // 2)) // mult * mult))
        b.append(x)
    return b


JOIN_TYPES = [(INNER_JOIN, False), (INNER_JOIN, True), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)]


# every join type on the one-table path (build side below 2^18 rows: ordered compare); two on the partitioned path (multiset)
JOIN_CASES = [(jt, oir, 0) for jt, oir in JOIN_TYPES] + [(INNER_JOIN, False, 1), (RIGHT_OUTER_JOIN, True, 1)]


@pytest.mark.parametrize("jt,oir,big", JOIN_CASES)
def test_join_string_key(lib, jt, oir, big):
    nb = (1 << 18) + 4000 if big else 6000
    rng = np.random.default_rng(nb + 10 * jt + oir)
    npr = 40000
    words = max(nb // 3, 10)
    b = [Column(BYTES, vocab(rng, words, 0.05, nb)), Column(INT64, np.arange(nb))]
    p = [Column(INT64, np.arange(npr)), Column(BYTES, vocab(rng, words + words // 5, 0.05, npr)), Column(BYTES, vocab(rng, 50, 0.2, npr, 90))]
    bt, pt = [BYTES, INT64], [INT64, BYTES, BYTES]
    got = join_device(lib, jt, oir, bt, b, pt, p, [0], [1], ragged_bounds(rng, nb, nb // 3), ragged_bounds(rng, npr, 7000, 1), batch=4096)
    want = O.hash_join(jt, oir, bt, b, pt, p, [0], [1])
    if nb < (1 << 18):
        assert_same_ordered(got, want)   # one table: (probe row, build insertion) order
    else:
        assert_same_multiset(got, want)


@pytest.mark.parametrize("jt,oir,big", JOIN_CASES)
def test_join_bigint_varchar_keys(lib, jt, oir, big):
    """the reference's default key {BIGINT, VARCHAR}; string payloads on both sides"""
    nb = (1 << 18) + 1000 if big else 5000
    rng = np.random.default_rng(3 * nb + 10 * jt + oir)
    npr = 30000
    bk = rng.integers(0, nb // 2, nb)
    b = [Column(INT64, bk, rng.random(nb) > 0.03), Column(BYTES, [cell_of(rng, int(v) % 40) if rng.random() > 0.03 else None for v in bk]),
         Column(BYTES, vocab(rng, 300, 0.1, nb, 80))]
    pk = rng.integers(0, nb // 2 + 500, npr)
    p = [Column(INT64, pk), Column(BYTES, [cell_of(rng, int(v) % 40 + (1 if rng.random() < 0.1 else 0)) for v in pk]),
         Column(BYTES, vocab(rng, 70, 0.1, npr, 70)), Column(INT64, np.arange(npr))]
    bt, pt = [INT64, BYTES, BYTES], [INT64, BYTES, BYTES, INT64]
    got = join_device(lib, jt, oir, bt, b, pt, p, [0, 1], [0, 1], ragged_bounds(rng, nb, nb // 4), ragged_bounds(rng, npr, 9000, 1))
    want = O.hash_join(jt, oir, bt, b, pt, p, [0, 1], [0, 1])
    if nb < (1 << 18):
        assert_same_ordered(got, want)
    else:
        assert_same_multiset(got, want)


# ------------------------------------------------------------------------------------------------------------- aggregation
def agg_outputs(lib, h, types):
    out = (L.TQColumn * len(types))()
    n, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_agg_next_device(h, out, C.byref(n), C.byref(eof)))
    got = lent_to_host(types, out, n.value)
    L.check(lib.tq_agg_next_device(h, out, C.byref(n), C.byref(eof)))
    assert n.value == 0 and eof.value == 1
    return got


def agg_device(lib, types, cols, group_by, funcs, bounds):
    fa = (L.TQAggFunc * len(funcs))(*[L.TQAggFunc(f, a) for f, a in funcs])
    d = L.TQAggDesc(len(types), i32(types), len(group_by), i32(group_by), len(funcs), fa, 0)
    h = C.c_void_p()
    L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
    for dcs, arr in device_pieces(cols, bounds):
        L.check(lib.tq_agg_put(h, arr, L.TQ_MEM_DEVICE))
        scribble_cells(lib, dcs)
        free_all(dcs)                # the put has finished reading the chunk
    L.check(lib.tq_agg_eof(h))
    got = agg_outputs(lib, h, [O.agg_out_type(f, types[a] if a >= 0 else INT64) for f, a in funcs])
    L.check(lib.tq_agg_destroy(h))
    return got


def test_agg_string_group_by_and_arguments(lib):
    rng = np.random.default_rng(5)
    n = 120000
    g = Column(BYTES, vocab(rng, 1500, 0.03, n))
    s = Column(BYTES, vocab(rng, 4000, 0.2, n, 120))
    x = Column(INT64, rng.integers(-1000, 1000, n), rng.random(n) > 0.1)
    types, cols = [BYTES, BYTES, INT64], [g, s, x]
    funcs = [(AGG_COUNT, 1), (AGG_MAX, 1), (AGG_MIN, 1), (AGG_FIRSTROW, 0), (AGG_COUNT, -1), (AGG_SUM, 2)]
    got = agg_device(lib, types, cols, [0], funcs, ragged_bounds(rng, n, 20000, 1))
    rc, want = O.hash_agg(types, cols, [0], funcs)
    assert rc == 0
    assert_same_multiset(got, want)
    # several GROUP BY items, one of them a string; scalar aggregation over strings
    for gb, fs in (([2, 0], [(AGG_MAX, 1), (AGG_FIRSTROW, 0), (AGG_FIRSTROW, 2), (AGG_COUNT, 1)]), ([], [(AGG_MAX, 1), (AGG_MIN, 1), (AGG_COUNT, 1)])):
        got = agg_device(lib, types, cols, gb, fs, ragged_bounds(rng, n, 30000, 1))
        rc, want = O.hash_agg(types, cols, gb, fs)
        assert rc == 0
        assert_same_multiset(got, want)


def test_agg_final_mode_string_partial_columns(lib):
    """FinalMode: partial rows (COUNT, MAX, MIN, group value) with string partial columns, fed as device chunks"""
    rng = np.random.default_rng(6)
    n = 30000
    cnt = Column(INT64, rng.integers(0, 50, n))
    mx = Column(BYTES, vocab(rng, 900, 0.1, n, 70))
    mn = Column(BYTES, vocab(rng, 900, 0.1, n))
    key = Column(BYTES, vocab(rng, 700, 0.02, n))
    types, cols = [INT64, BYTES, BYTES, BYTES], [cnt, mx, mn, key]
    ff = [(AGG_COUNT, 0, -1), (AGG_MAX, 1, -1), (AGG_MIN, 2, -1), (AGG_FIRSTROW, 3, -1)]
    fa = (L.TQAggFinalFunc * len(ff))(*[L.TQAggFinalFunc(*f) for f in ff])
    d = L.TQAggFinalDesc(len(types), i32(types), 1, i32([3]), len(ff), fa, 0)
    h = C.c_void_p()
    L.check(lib.tq_agg_create_final(C.byref(d), C.byref(h)))
    for dcs, arr in device_pieces(cols, ragged_bounds(rng, n, 6000, 1)):
        L.check(lib.tq_agg_put(h, arr, L.TQ_MEM_DEVICE))
        scribble_cells(lib, dcs)
        free_all(dcs)
    L.check(lib.tq_agg_eof(h))
    got = agg_outputs(lib, h, [INT64, BYTES, BYTES, BYTES])
    L.check(lib.tq_agg_destroy(h))
    rc, want = O.hash_agg_final(types, cols, [3], ff)
    assert rc == 0
    assert_same_multiset(got, want)


# ------------------------------------------------------------------------------------------------------------- sort / TopN
def sort_device(lib, types, cols, by, bounds, off=0, cnt=-1, host_next=False):
    d = L.TQSortDesc(len(types), i32(types), len(by), i32([c for c, _ in by]), i32([1 if x else 0 for _, x in by]), off, cnt)
    h = C.c_void_p()
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    for dcs, arr in device_pieces(cols, bounds):
        L.check(lib.tq_sort_put(h, arr, L.TQ_MEM_DEVICE))
        scribble_cells(lib, dcs)
        free_all(dcs)                # the call has copied what it keeps
    L.check(lib.tq_sort_eof(h))
    n, eof = C.c_int64(0), C.c_int32(0)
    if host_next:
        cap = 1 << 20
        nb = (C.c_int64 * len(types))()
        L.check(lib.tq_sort_next_bytes(h, cap, nb))
        res = [VarColumn.empty(BYTES, cap, int(nb[i])) if t == BYTES else Column.empty(t, cap) for i, t in enumerate(types)]
        L.check(lib.tq_sort_next(h, cap, tq_array(res, cap), C.byref(n), C.byref(eof)))
        got = Chunk([c.head(n.value) if c.tp == BYTES else Column(c.tp, c.values[: n.value].copy(), c.not_null()[: n.value].copy()) for c in res])
    else:
        out = (L.TQColumn * len(types))()
        L.check(lib.tq_sort_next_device(h, out, C.byref(n), C.byref(eof)))
        got = lent_to_host(types, out, n.value)
        L.check(lib.tq_sort_next_device(h, out, C.byref(n), C.byref(eof)))
        assert n.value == 0 and eof.value == 1
    L.check(lib.tq_sort_destroy(h))
    return got


def sort_body(lib, n, piece):
    rng = np.random.default_rng(n + piece)
    s = vocab(rng, max(n // 4, 5), 0.08, n)
    # the last piece holds the longest cells, so the number of string key words grows with the last put
    last = (n - 1) // piece * piece
    for i in range(last, n, 3):
        s[i] = (s[i] or b"z") + b"~" * int(rng.integers(60, 140))
    types = [BYTES, INT64, BYTES]
    cols = [Column(BYTES, s), Column(INT64, rng.integers(0, 5, n)), Column(BYTES, vocab(rng, 30, 0.1, n, 40))]
    bounds = list(range(0, n, piece)) + [n]
    for by in ([(0, False)], [(0, True)], [(1, False), (0, True)], [(2, False), (0, False)]):
        assert_same_ordered(sort_device(lib, types, cols, by, bounds), O.sort(types, cols, by))
    assert_same_ordered(sort_device(lib, types, cols, [(0, True), (1, False)], bounds, 3, 100), O.sort(types, cols, [(0, True), (1, False)], 3, 100))
    assert_same_ordered(sort_device(lib, types, cols, [(0, False)], bounds, host_next=True), O.sort(types, cols, [(0, False)]))   # lazy host copy


@pytest.mark.parametrize("n,piece", [(1, 100), (3001, 700), (60001, 9000)])
def test_sort_string_by_items(lib, n, piece):
    sort_body(lib, n, piece)


# ------------------------------------------------------------------------------------------------------------- merge join
def mjoin_device(lib, jt, oir, it, inner, ot, outer, ik, ok, ibounds, obounds):
    md = L.TQMJoinDesc(jt, 1 if oir else 0, len(it), i32(it), len(ot), i32(ot), len(ik), i32(ik), i32(ok), None, None)
    h = C.c_void_p()
    L.check(lib.tq_mjoin_create(C.byref(md), C.byref(h)))
    for dcs, arr in device_pieces(inner, ibounds):
        L.check(lib.tq_mjoin_put_inner(h, arr, L.TQ_MEM_DEVICE))
        scribble_cells(lib, dcs)
        free_all(dcs)
    for dcs, arr in device_pieces(outer, obounds):
        L.check(lib.tq_mjoin_put_outer(h, arr, None, L.TQ_MEM_DEVICE))
        scribble_cells(lib, dcs)
        free_all(dcs)
    L.check(lib.tq_mjoin_finish(h))
    types = (it + ot) if oir else (ot + it)
    out = (L.TQColumn * len(types))()
    n, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_mjoin_next_device(h, out, C.byref(n), C.byref(eof)))
    got = lent_to_host(types, out, n.value)
    L.check(lib.tq_mjoin_destroy(h))
    return got


def merge_join_body(lib, ni, no):
    rng = np.random.default_rng(ni + no)
    it, ot = [BYTES, INT64], [INT64, BYTES, BYTES]
    inner = O.sort(it, [Column(BYTES, vocab(rng, 300, 0.05, ni)), Column(INT64, np.arange(ni))], [(0, False)]).cols
    outer = O.sort(ot, [Column(INT64, np.arange(no)), Column(BYTES, vocab(rng, 340, 0.05, no)), Column(BYTES, vocab(rng, 20, 0.3, no, 80))],
                   [(1, False)]).cols
    for jt, oir in ((INNER_JOIN, False), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)):
        got = mjoin_device(lib, jt, oir, it, inner, ot, outer, [0], [1], ragged_bounds(rng, ni, ni // 3, 1), ragged_bounds(rng, no, no // 4, 1))
        assert_same_ordered(got, O.merge_join(jt, oir, it, inner, ot, outer, [0], [1]))


def test_merge_join_string_keys(lib):
    merge_join_body(lib, 4000, 6000)


# ------------------------------------------------------------------------------------------------------------- chains
def decode_pieces(types, cols, rows_per_chunk):
    """encode the table as wire chunks and decode each one into HBM"""
    n = cols[0].length
    for lo in range(0, n, rows_per_chunk):
        hi = min(n, lo + rows_per_chunk)
        yield DeviceChunk().decode(encode_chunk(types, [piece(c, lo, hi) for c in cols]), types)


def test_chain_decode_join_sort_merge_join(lib):
    """{BIGINT, VARCHAR} chunks -> tq_chunk_decode_device -> hash join on {0, 1} -> sort by the string -> merge join;
    every hand-over in HBM"""
    rng = np.random.default_rng(21)
    nb, npr = 20000, 60000
    bk = rng.permutation(nb)
    bt = [INT64, BYTES]
    b = [Column(INT64, bk), Column(BYTES, [cell_of(rng, int(v)) + b"/%d" % (v % 997) for v in bk])]
    pk = rng.integers(0, nb + 2000, npr)
    pt = [INT64, BYTES, INT64]
    p = [Column(INT64, pk), Column(BYTES, [cell_of(rng, int(v)) + b"/%d" % (v % 997) if rng.random() > 0.05 else b"x" for v in pk]),
         Column(INT64, np.arange(npr))]
    d = L.TQJoinDesc(INNER_JOIN, 1, 2, i32(bt), 3, i32(pt), 2, i32([0, 1]), i32([0, 1]), 0, 0)
    hj = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(hj)))
    kept = []
    for dc in decode_pieces(bt, b, 7000):
        L.check(lib.tq_join_put_build(hj, dc.tq_cols, L.TQ_MEM_DEVICE))
        kept.append(dc)
    L.check(lib.tq_join_finalize_build(hj))
    jt5 = bt + pt                                           # (B.k, B.s, P.k, P.s, P.id)
    sd = L.TQSortDesc(5, i32(jt5), 2, i32([1, 4]), i32([0, 0]), 0, -1)
    hs = C.c_void_p()
    L.check(lib.tq_sort_create(C.byref(sd), C.byref(hs)))
    joined = (L.TQColumn * 5)()
    n, eof = C.c_int64(0), C.c_int32(0)
    parts = []

    def feed_sort():
        while True:
            L.check(lib.tq_join_next_device(hj, joined, C.byref(n), C.byref(eof)))
            if n.value == 0:
                return
            parts.append(lent_to_host(jt5, joined, n.value))
            L.check(lib.tq_sort_put(hs, joined, L.TQ_MEM_DEVICE))   # the lent batch goes straight on

    dp = DeviceChunk()
    for lo in range(0, npr, 16000):
        dp.decode(encode_chunk(pt, [piece(c, lo, min(npr, lo + 16000)) for c in p]), pt)
        L.check(lib.tq_join_put_probe(hj, dp.tq_cols, None, L.TQ_MEM_DEVICE))
        feed_sort()
    L.check(lib.tq_join_probe_eof(hj))
    feed_sort()
    dp.free()
    for dc in kept:
        dc.free()
    L.check(lib.tq_join_destroy(hj))
    want_join = O.hash_join(INNER_JOIN, True, bt, b, pt, p, [0, 1], [0, 1])
    assert_same_multiset(Chunk.concat(parts, jt5), want_join)
    L.check(lib.tq_sort_eof(hs))
    sorted_cols = (L.TQColumn * 5)()
    ns = C.c_int64(0)
    L.check(lib.tq_sort_next_device(hs, sorted_cols, C.byref(ns), C.byref(eof)))
    want_sorted = O.sort(jt5, want_join.cols, [(1, False), (4, False)])   # P.id is unique: the order is total
    assert_same_ordered(lent_to_host(jt5, sorted_cols, ns.value), want_sorted)
    # MergeJoinExec: inner child = the build table sorted by its string (device chunks), outer child = the sorted join rows
    inner_sorted = O.sort(bt, b, [(1, False)])
    md = L.TQMJoinDesc(LEFT_OUTER_JOIN, 0, 2, i32(bt), 5, i32(jt5), 1, i32([1]), i32([1]), None, None)
    hm = C.c_void_p()
    L.check(lib.tq_mjoin_create(C.byref(md), C.byref(hm)))
    for dcs, arr in device_pieces(inner_sorted.cols, [0, 5000, 12000, nb]):
        L.check(lib.tq_mjoin_put_inner(hm, arr, L.TQ_MEM_DEVICE))
        free_all(dcs)
    L.check(lib.tq_mjoin_put_outer(hm, sorted_cols, None, L.TQ_MEM_DEVICE))
    L.check(lib.tq_sort_destroy(hs))
    L.check(lib.tq_mjoin_finish(hm))
    mj = (L.TQColumn * 7)()
    nm = C.c_int64(0)
    L.check(lib.tq_mjoin_next_device(hm, mj, C.byref(nm), C.byref(eof)))
    got_mj = lent_to_host(jt5 + bt, mj, nm.value)
    L.check(lib.tq_mjoin_destroy(hm))
    assert_same_ordered(got_mj, O.merge_join(LEFT_OUTER_JOIN, False, bt, inner_sorted.cols, jt5, want_sorted.cols, [1], [1]))


def test_chain_decode_group_by_string_then_topn(lib):
    """decode -> string GROUP BY -> tq_agg_next_device -> TopN, in HBM"""
    rng = np.random.default_rng(22)
    n = 200000
    at = [BYTES, INT64]
    cols = [Column(BYTES, vocab(rng, 3000, 0.01, n)), Column(INT64, rng.integers(0, 100, n), rng.random(n) > 0.1)]
    funcs = [(AGG_FIRSTROW, 0), (AGG_COUNT, -1), (AGG_MAX, 1)]
    fa = (L.TQAggFunc * 3)(*[L.TQAggFunc(f, a) for f, a in funcs])
    ad = L.TQAggDesc(2, i32(at), 1, i32([0]), 3, fa, 3000)
    ha = C.c_void_p()
    L.check(lib.tq_agg_create(C.byref(ad), C.byref(ha)))
    dc = DeviceChunk()
    for lo in range(0, n, 50000):
        dc.decode(encode_chunk(at, [piece(c, lo, min(n, lo + 50000)) for c in cols]), at)
        L.check(lib.tq_agg_put(ha, dc.tq_cols, L.TQ_MEM_DEVICE))
    dc.free()
    L.check(lib.tq_agg_eof(ha))
    ot = [BYTES, INT64, INT64]
    lent = (L.TQColumn * 3)()
    ng, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_agg_next_device(ha, lent, C.byref(ng), C.byref(eof)))
    rc, want_agg = O.hash_agg(at, cols, [0], funcs)
    assert rc == 0
    got_agg = lent_to_host(ot, lent, ng.value)
    assert_same_multiset(got_agg, want_agg)
    by = [(1, True), (0, False)]                           # the group value is unique: the order is total
    sd = L.TQSortDesc(3, i32(ot), 2, i32([1, 0]), i32([1, 0]), 2, 25)
    hs = C.c_void_p()
    L.check(lib.tq_sort_create(C.byref(sd), C.byref(hs)))
    L.check(lib.tq_sort_put(hs, lent, L.TQ_MEM_DEVICE))
    L.check(lib.tq_agg_destroy(ha))
    L.check(lib.tq_sort_eof(hs))
    top = (L.TQColumn * 3)()
    nt = C.c_int64(0)
    L.check(lib.tq_sort_next_device(hs, top, C.byref(nt), C.byref(eof)))
    assert_same_ordered(lent_to_host(ot, top, nt.value), O.sort(ot, got_agg.cols, by, 2, 25))
    assert_same_ordered(lent_to_host(ot, top, nt.value), O.sort(ot, want_agg.cols, by, 2, 25))
    L.check(lib.tq_sort_destroy(hs))


# ------------------------------------------------------------------------------------------------------------- rules
def sort_mjoin_rules(lib):
    """FLOAT device columns are refused, host and device chunks do not mix, a var-len device column needs offsets, and bad
    device offsets are refused without changing what the handle holds"""
    s = DeviceVarColumn.from_host(Column(BYTES, [b"b", None, b"a"]), 3)
    i = DeviceColumn.from_host(Column(INT64, [3, 1, 2]))
    # sort: FLOAT from HBM is still refused
    h = C.c_void_p()
    d = L.TQSortDesc(2, i32([BYTES, FLOAT32]), 1, i32([0]), i32([0]), 0, -1)
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    assert lib.tq_sort_put(h, (L.TQColumn * 2)(s.tq(), i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_UNSUPPORTED_TYPE
    L.check(lib.tq_sort_destroy(h))
    # sort: no offsets; host after device; offsets that go backwards
    d = L.TQSortDesc(2, i32([BYTES, INT64]), 1, i32([0]), i32([0]), 0, -1)
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    no_off = s.tq()
    no_off.offsets = None
    assert lib.tq_sort_put(h, (L.TQColumn * 2)(no_off, i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_INVALID_ARG
    L.check(lib.tq_sort_put(h, (L.TQColumn * 2)(s.tq(), i.tq()), L.TQ_MEM_DEVICE))
    bad = DeviceColumn.from_host(Column(INT64, [0, 5, 3, 4]))      # offsets 0, 5, 3, 4
    t = s.tq()
    t.offsets = bad._data.value
    assert lib.tq_sort_put(h, (L.TQColumn * 2)(t, i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_INVALID_ARG
    host = [Column(BYTES, [b"c"]), Column(INT64, [9])]
    assert lib.tq_sort_put(h, tq_array(host), L.TQ_MEM_HOST) == L.TQ_ERR_STATE
    L.check(lib.tq_sort_eof(h))
    out = (L.TQColumn * 2)()
    n, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_sort_next_device(h, out, C.byref(n), C.byref(eof)))
    assert lent_to_host([BYTES, INT64], out, n.value).rows() == [(None, 1), (b"a", 2), (b"b", 3)]
    L.check(lib.tq_sort_destroy(h))
    # merge join: the same rules per child
    md = L.TQMJoinDesc(0, 0, 2, i32([BYTES, FLOAT32]), 2, i32([BYTES, INT64]), 1, i32([0]), i32([0]), None, None)
    L.check(lib.tq_mjoin_create(C.byref(md), C.byref(h)))
    assert lib.tq_mjoin_put_inner(h, (L.TQColumn * 2)(s.tq(), i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_UNSUPPORTED_TYPE
    assert lib.tq_mjoin_put_outer(h, (L.TQColumn * 2)(no_off, i.tq()), None, L.TQ_MEM_DEVICE) == L.TQ_ERR_INVALID_ARG
    L.check(lib.tq_mjoin_put_outer(h, (L.TQColumn * 2)(s.tq(), i.tq()), None, L.TQ_MEM_DEVICE))
    assert lib.tq_mjoin_put_outer(h, tq_array(host), None, L.TQ_MEM_HOST) == L.TQ_ERR_STATE
    L.check(lib.tq_mjoin_destroy(h))
    for x in (s, i, bad):
        x.free()


def test_device_varlen_rules(lib):
    sort_mjoin_rules(lib)
    s = DeviceVarColumn.from_host(Column(BYTES, [b"b", None, b"a"]), 3)
    i = DeviceColumn.from_host(Column(INT64, [3, 1, 2]))
    no_off = s.tq()
    no_off.offsets = None
    h = C.c_void_p()
    # hash join: FLOAT from HBM refused on both sides, var-len needs offsets
    d = L.TQJoinDesc(0, 0, 2, i32([BYTES, FLOAT32]), 2, i32([BYTES, INT64]), 1, i32([0]), i32([0]), 0, 0)
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    assert lib.tq_join_put_build(h, (L.TQColumn * 2)(s.tq(), i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_UNSUPPORTED_TYPE
    assert lib.tq_join_put_build(h, (L.TQColumn * 2)(no_off, i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_INVALID_ARG
    L.check(lib.tq_join_destroy(h))
    d = L.TQJoinDesc(0, 0, 2, i32([BYTES, INT64]), 2, i32([BYTES, FLOAT32]), 1, i32([0]), i32([0]), 0, 0)
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    L.check(lib.tq_join_put_build(h, (L.TQColumn * 2)(s.tq(), i.tq()), L.TQ_MEM_DEVICE))
    L.check(lib.tq_join_finalize_build(h))
    assert lib.tq_join_put_probe(h, (L.TQColumn * 2)(s.tq(), i.tq()), None, L.TQ_MEM_DEVICE) == L.TQ_ERR_UNSUPPORTED_TYPE
    assert lib.tq_join_put_probe(h, (L.TQColumn * 2)(no_off, i.tq()), None, L.TQ_MEM_DEVICE) == L.TQ_ERR_INVALID_ARG
    L.check(lib.tq_join_destroy(h))
    # build chunks are all host or all device, as before
    d = L.TQJoinDesc(0, 0, 2, i32([BYTES, INT64]), 2, i32([BYTES, INT64]), 1, i32([0]), i32([0]), 0, 0)
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    L.check(lib.tq_join_put_build(h, tq_array([Column(BYTES, [b"a"]), Column(INT64, [1])]), L.TQ_MEM_HOST))
    assert lib.tq_join_put_build(h, (L.TQColumn * 2)(s.tq(), i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_INVALID_ARG
    L.check(lib.tq_join_destroy(h))
    # aggregation: FLOAT from HBM refused, var-len needs offsets
    fa = (L.TQAggFunc * 1)(L.TQAggFunc(AGG_COUNT, 1))
    ad = L.TQAggDesc(2, i32([BYTES, FLOAT32]), 1, i32([0]), 1, fa, 0)
    L.check(lib.tq_agg_create(C.byref(ad), C.byref(h)))
    assert lib.tq_agg_put(h, (L.TQColumn * 2)(s.tq(), i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_UNSUPPORTED_TYPE
    L.check(lib.tq_agg_destroy(h))
    ad = L.TQAggDesc(2, i32([BYTES, INT64]), 1, i32([0]), 1, fa, 0)
    L.check(lib.tq_agg_create(C.byref(ad), C.byref(h)))
    assert lib.tq_agg_put(h, (L.TQColumn * 2)(no_off, i.tq()), L.TQ_MEM_DEVICE) == L.TQ_ERR_INVALID_ARG
    L.check(lib.tq_agg_destroy(h))
    s.free()
    i.free()
