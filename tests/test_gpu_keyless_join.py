"""The key-less hash join on the device (tq_join_desc.n_keys == 0): ordered parity with the oracle, 64-bit pair spaces,
lazily built result batches, errors and warnings of the conditions, and the C-ABI corners."""
import ctypes as C

import numpy as np
import pytest

from join_program_oracle import OracleError
from keyless_oracle import keyless_hash_join, keyless_join_with_program, nested_loop
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, FLOAT32, FLOAT64, INT64, Chunk, Column, DeviceColumn, device_to_host, device_var_to_host
from tinysql_b200.executor import INNER_JOIN, LEFT_OUTER_JOIN, RIGHT_OUTER_JOIN, HashJoinExec, MockDataSource
from tinysql_b200.expression import Col, Const, Func, JoinProgram
from util import assert_same_ordered

pytestmark = pytest.mark.gpu
LT, GE = 0, 3
SHAPES = [(INNER_JOIN, False), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)]


def _sides(rng, nb, npr, indirect=True):
    bt = [INT64, BYTES, FLOAT32] if indirect else [INT64, INT64]
    bc = [Column(INT64, rng.integers(0, 50, nb), rng.random(nb) > 0.1)]
    bc += [Column(BYTES, [None if rng.random() < 0.1 else b"s%d" % rng.integers(0, 1000) for _ in range(nb)]),
           Column(FLOAT32, rng.random(nb).astype(np.float32), rng.random(nb) > 0.2)] if indirect else [Column(INT64, np.arange(nb))]
    pt = [INT64, FLOAT64]
    pc = [Column(INT64, rng.integers(0, 50, npr), rng.random(npr) > 0.1), Column(FLOAT64, rng.random(npr))]
    return bt, bc, pt, pc


def _run_exec(bt, bc, pt, pc, jt, oir, sel=None, dflt=None, conds=(), program=(), batch=0, chunk=1024):
    flt = None if sel is None else (lambda chk, _s=iter([np.asarray(sel[i:i + chunk], dtype=np.uint8) for i in range(0, len(sel), chunk)]): next(_s))
    e = HashJoinExec(MockDataSource(pt, pc, chunk), MockDataSource(bt, bc, chunk), [], [], jt, oir, outer_filter=flt, probe_batch_rows=batch,
                     other_conditions=conds, other_program=program, default_inner=dflt)
    e.Open()
    try:
        got = e.drain()
        return got, e.warnings
    finally:
        e.Close()


def _create(lib, jt, oir, bt, pt, batch=0, dflt=None):
    bta, pta = (C.c_int32 * len(bt))(*bt), (C.c_int32 * len(pt))(*pt)
    d = L.TQJoinDesc(jt, 1 if oir else 0, len(bt), bta, len(pt), pta, 0, None, None, batch, 0)
    keep = [bta, pta]
    if dflt is not None:
        keep += [(C.c_uint64 * len(bt))(*[0 if v is None else int(v) for v in dflt]), (C.c_uint8 * len(bt))(*[v is not None for v in dflt])]
        d.default_inner_bits, d.default_inner_not_null = keep[-2], keep[-1]
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    return h, keep


def _dev_cols(cols):
    return [DeviceColumn.from_host(c) for c in cols]


def _drain_device(lib, h, types):
    """tq_join_next_device until eof -> Chunk"""
    chunks = []
    arr = (L.TQColumn * len(types))()
    n, eof = C.c_int64(0), C.c_int32(0)
    while True:
        L.check(lib.tq_join_next_device(h, arr, C.byref(n), C.byref(eof)))
        if n.value:
            chunks.append(Chunk([device_var_to_host(arr[c].data, arr[c].offsets, arr[c].null_bitmap, n.value) if t == BYTES
                                 else device_to_host(t, arr[c].data, arr[c].null_bitmap, n.value) for c, t in enumerate(types)]))
        elif eof.value:
            return Chunk.concat(chunks, types)


@pytest.mark.parametrize("jt,oir", SHAPES)
@pytest.mark.parametrize("form", ["none", "conds", "program"])
@pytest.mark.parametrize("nb", [0, 33, 1000])
def test_keyless_exec_host_chunks(lib, jt, oir, form, nb):
    rng = np.random.default_rng(nb + 3 * jt + (form == "conds") * 7 + (form == "program") * 13)
    npr = 2500
    bt, bc, pt, pc = _sides(rng, nb, npr)
    sel = rng.random(npr) > 0.2
    dflt = [7, None, None] if jt != INNER_JOIN else None
    n_left = len(bt) if oir else len(pt)
    bvo, pvo = (0, n_left) if oir else (n_left, 0)
    conds = [(LT, bvo, pvo)] if form == "conds" else []
    program = [Func("ge", Func("plus", Col(bvo), Col(pvo)), Const(60))] if form == "program" else []
    got, warn = _run_exec(bt, bc, pt, pc, jt, oir, sel, dflt, conds, program)
    if form == "program":
        want, wwarn = keyless_join_with_program(jt, oir, bt, bc, pt, pc, program, sel, dflt)
        assert warn == wwarn
    else:
        want = keyless_hash_join(jt, oir, bt, bc, pt, pc, sel, conds, dflt)
    assert_same_ordered(got, want)


@pytest.mark.parametrize("jt,oir", SHAPES)
@pytest.mark.parametrize("form", ["none", "conds"])
def test_keyless_device_puts(lib, jt, oir, form):
    rng = np.random.default_rng(40 + jt + (form == "conds"))
    nb, npr = 700, 3000
    bt = [INT64, BYTES]
    bc = [Column(INT64, rng.integers(0, 50, nb), rng.random(nb) > 0.1), Column(BYTES, [None if rng.random() < 0.1 else b"b%d" % i for i in range(nb)])]
    pt = [INT64, BYTES]
    pc = [Column(INT64, rng.integers(0, 50, npr), rng.random(npr) > 0.1), Column(BYTES, [b"p%d" % i for i in range(npr)])]
    sel = (rng.random(npr) > 0.2).astype(np.uint8)
    n_left = len(bt) if oir else len(pt)
    conds = [(LT, 0, n_left) if oir else (LT, n_left, 0)] if form == "conds" else []
    h, keep = _create(lib, jt, oir, bt, pt, batch=4096)
    try:
        if conds:
            arr = (L.TQJoinCond * 1)(L.TQJoinCond(conds[0][0], conds[0][1], conds[0][2], 0, 0))
            L.check(lib.tq_join_set_other_conditions(h, 1, arr))
        dbc = _dev_cols(bc)
        L.check(lib.tq_join_put_build(h, (L.TQColumn * 2)(*[d.tq() for d in dbc]), L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        for d in dbc:
            d.free()   # a single device build chunk is lent only until finalize_build
        for lo in range(0, npr, 1000):
            dpc = _dev_cols([c.slice(lo, lo + 1000) for c in pc])
            s = np.ascontiguousarray(sel[lo:lo + 1000])
            L.check(lib.tq_join_put_probe(h, (L.TQColumn * 2)(*[d.tq() for d in dpc]), s.ctypes.data, L.TQ_MEM_DEVICE))
            for d in dpc:
                d.free()   # the probe rows are copied: the caller's buffers are free once the call returns
        L.check(lib.tq_join_probe_eof(h))
        types = bt + pt if oir else pt + bt
        got = _drain_device(lib, h, types)
    finally:
        lib.tq_join_destroy(h)
    assert_same_ordered(got, keyless_hash_join(jt, oir, bt, bc, pt, pc, sel, conds))


@pytest.mark.parametrize("batch", [64, 1024])
@pytest.mark.parametrize("form", ["none", "conds"])
def test_keyless_pairs_span_result_batches(lib, batch, form):
    """build 5000 x probe 300: one probe row's pairs fill many result batches"""
    rng = np.random.default_rng(batch)
    nb, npr = 5000, 300
    bc = [Column(INT64, np.arange(nb)), Column(INT64, rng.integers(0, 1 << 40, nb), rng.random(nb) > 0.3)]
    pc = [Column(INT64, rng.integers(-10, 2 * nb, npr)), Column(INT64, np.arange(npr))]
    conds = [(LT, 2, 0)] if form == "conds" else []   # B.v < P.v over left = probe ++ right = build
    got, _ = _run_exec([INT64, INT64], bc, [INT64, INT64], pc, LEFT_OUTER_JOIN, False, conds=conds, batch=batch)
    pv = pc[0].values
    want = nested_loop(LEFT_OUTER_JOIN, False, bc, pc, None, (lambda pi, bi: bc[0].values[bi] < pv[pi]) if conds else None)
    assert got.num_rows() == want.num_rows() == (npr * nb if not conds else int(np.maximum(np.minimum(pv, nb), 1).sum()))
    assert_same_ordered(got, want)


def test_keyless_64bit_pair_space(lib):
    """probe 10^6 x build 5000 = 5e9 pairs under B.v < P.v, B.v = 0..B-1: probe row i keeps min(max(P.v_i, 0), B) rows"""
    rng = np.random.default_rng(5)
    nb, npr = 5000, 1_000_000
    bc = [Column(INT64, np.arange(nb))]
    pv = rng.integers(-5, 26, npr)
    pv[rng.choice(npr, 200, replace=False)] = rng.integers(nb - 3, nb + 1000, 200)   # a few rows keep (almost) the whole build side
    pc = [Column(INT64, pv), Column(INT64, np.arange(npr))]
    h, keep = _create(lib, INNER_JOIN, False, [INT64], [INT64, INT64])
    try:
        arr = (L.TQJoinCond * 1)(L.TQJoinCond(LT, 2, 0, 0, 0))
        L.check(lib.tq_join_set_other_conditions(h, 1, arr))
        dbc = _dev_cols(bc)
        L.check(lib.tq_join_put_build(h, (L.TQColumn * 1)(*[d.tq() for d in dbc]), L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        dpc = _dev_cols(pc)
        L.check(lib.tq_join_put_probe(h, (L.TQColumn * 2)(*[d.tq() for d in dpc]), None, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_probe_eof(h))
        got = _drain_device(lib, h, [INT64, INT64, INT64])
        for d in dbc + dpc:
            d.free()
    finally:
        lib.tq_join_destroy(h)
    want_cnt = np.minimum(np.maximum(pv, 0), nb)
    assert got.num_rows() == int(want_cnt.sum())
    rid = got.cols[1].values
    assert np.array_equal(np.bincount(rid, minlength=npr), want_cnt)
    assert np.all(np.diff(rid) >= 0)   # probe row ascending ...
    start = np.repeat(np.cumsum(want_cnt) - want_cnt, want_cnt)
    assert np.array_equal(got.cols[2].values, np.arange(got.num_rows()) - start)   # ... build insertion ascending
    sample = rng.choice(npr, 1000, replace=False)
    assert np.array_equal(got.cols[0].values[np.isin(rid, sample)], np.repeat(pv[np.sort(sample)], want_cnt[np.sort(sample)]))


def test_keyless_result_batches_are_lazy(lib):
    """a 10^6 x 10^6 cross join: a few result batches, then destroy — nothing of the 10^12 rows is built ahead"""
    import torch
    n = 1_000_000
    batch = 1 << 20
    h, keep = _create(lib, INNER_JOIN, False, [INT64], [INT64], batch=batch)
    stats = (C.c_int64 * 8)()
    try:
        db, dp = DeviceColumn.from_host(Column(INT64, np.arange(n))), DeviceColumn.from_host(Column(INT64, np.arange(n) * 3))
        L.check(lib.tq_join_put_build(h, (L.TQColumn * 1)(db.tq()), L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        L.check(lib.tq_join_put_probe(h, (L.TQColumn * 1)(dp.tq()), None, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_probe_eof(h))
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        arr = (L.TQColumn * 2)()
        rows, eof = C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_join_next_device(h, arr, C.byref(rows), C.byref(eof)))
        free1 = torch.cuda.mem_get_info()[0]
        assert rows.value == batch and not eof.value
        first = device_to_host(INT64, arr[0].data, arr[0].null_bitmap, 4), device_to_host(INT64, arr[1].data, arr[1].null_bitmap, 4)
        assert first[0].tolist() == [0, 0, 0, 0] and first[1].tolist() == [0, 1, 2, 3]
        for _ in range(3):
            L.check(lib.tq_join_next_device(h, arr, C.byref(rows), C.byref(eof)))
            assert rows.value == batch
        L.check(lib.tq_join_stats(h, stats))
        assert stats[0] == n and stats[1] == 0 and stats[2] == 0 and stats[3] == n
        assert stats[4] <= 6 * batch   # 4 batches handed out + at most one built ahead
        per_batch = batch * 2 * 8 + 2 * ((batch + 63) // 64) * 8
        assert free0 - free1 <= 3 * per_batch + (64 << 20), (free0 - free1, per_batch)
        db.free()
        dp.free()
    finally:
        lib.tq_join_destroy(h)


def test_keyless_next_is_lazy_through_exec(lib):
    """HashJoinExec.Next(1024) on a 10^6 x 10^6 cross join, then Close: stats[4] stays within 3 result batches"""
    n = 1_000_000
    e = HashJoinExec(MockDataSource([INT64], [Column(INT64, np.arange(n))], 1 << 17), MockDataSource([INT64], [Column(INT64, np.arange(n))], 1 << 17), [], [])
    e.Open()
    stats = (C.c_int64 * 8)()
    try:
        for _ in range(3):
            assert e.Next(1024).num_rows() == 1024
        L.check(lib.tq_join_stats(e.handle, stats))
        assert 0 < stats[4] <= 3 * (1 << 22)
    finally:
        e.Close()


def _overflow_sides():
    b = [Column(INT64, np.array([1, 2, (1 << 62), 3], dtype=np.int64))]
    p = [Column(INT64, np.array([5, (1 << 62), 7, 9], dtype=np.int64)), Column(INT64, np.arange(4))]
    return b, p


def test_keyless_overflow_and_narrowing(lib):
    b, p = _overflow_sides()
    plus = Func("plus", Col(0), Col(2))   # P.v + B.v: 2^62 + 2^62 overflows on the pair (probe 1, build 2)
    with pytest.raises(L.TQError) as ei:
        _run_exec([INT64], b, [INT64, INT64], p, INNER_JOIN, False, program=[Func("gt", plus, Const(0))])
    assert ei.value.status == L.TQ_ERR_OVERFLOW_BIGINT
    with pytest.raises(OracleError):
        keyless_join_with_program(INNER_JOIN, False, [INT64], b, [INT64, INT64], p, [Func("gt", plus, Const(0))])
    # an earlier FILTER item drops those pairs: nothing raises
    prog = [Func("lt", Col(0), Const(1 << 61)), Func("gt", plus, Const(0))]
    got, _ = _run_exec([INT64], b, [INT64, INT64], p, LEFT_OUTER_JOIN, False, program=prog)
    want, _ = keyless_join_with_program(LEFT_OUTER_JOIN, False, [INT64], b, [INT64, INT64], p, prog)
    assert_same_ordered(got, want)
    # unselected probe rows and an empty build side never run the conditions
    got, _ = _run_exec([INT64], b, [INT64, INT64], p, LEFT_OUTER_JOIN, False, sel=[1, 0, 1, 1], program=[Func("gt", plus, Const(0))])
    assert_same_ordered(got, keyless_join_with_program(LEFT_OUTER_JOIN, False, [INT64], b, [INT64, INT64], p, [Func("gt", plus, Const(0))], [1, 0, 1, 1])[0])
    empty = [Column(INT64, np.zeros(0, dtype=np.int64))]
    got, _ = _run_exec([INT64], empty, [INT64, INT64], p, LEFT_OUTER_JOIN, False, program=[Func("gt", plus, Const(0))])
    assert got.rows() == [(5, 0, None), (1 << 62, 1, None), (7, 2, None), (9, 3, None)]


def test_keyless_division_warnings(lib):
    rng = np.random.default_rng(9)
    nb, npr = 300, 4000
    bt, bc = [FLOAT64], [Column(FLOAT64, rng.integers(-2, 3, nb).astype(np.float64), rng.random(nb) > 0.1)]
    pt, pc = [FLOAT64, INT64], [Column(FLOAT64, rng.random(npr) * 10), Column(INT64, rng.integers(0, 100, npr))]
    sel = rng.random(npr) > 0.3
    prog = [Func("lt", Col(1), Const(30)), Func("gt", Func("div", Col(0, "real"), Col(2, "real")), Const(2.0, "real"))]
    got, warn = _run_exec(bt, bc, pt, pc, LEFT_OUTER_JOIN, False, sel=sel, program=prog)
    want, wwarn = keyless_join_with_program(LEFT_OUTER_JOIN, False, bt, bc, pt, pc, prog, sel)
    assert wwarn > 0 and warn == wwarn
    assert_same_ordered(got, want)


def test_keyless_abi(lib):
    # NULL key arrays; destroy right after create
    h, keep = _create(lib, INNER_JOIN, False, [INT64], [INT64, INT64])
    L.check(lib.tq_join_destroy(h))
    # put_probe_segments is refused before any device work; destroy in the middle of the stream
    h, keep = _create(lib, LEFT_OUTER_JOIN, False, [INT64], [INT64, INT64], batch=64)
    b = Column(INT64, np.arange(100))
    L.check(lib.tq_join_put_build(h, (L.TQColumn * 1)(b.tq()), L.TQ_MEM_HOST))
    L.check(lib.tq_join_finalize_build(h))
    cnt = (C.c_void_p * 1)(None)
    assert lib.tq_join_put_probe_segments(h, 1, (L.TQColumn * 2)(b.tq(), b.tq()), cnt, 100) == L.TQ_ERR_UNSUPPORTED_TYPE
    p = [Column(INT64, np.arange(1000)), Column(INT64, np.arange(1000))]
    L.check(lib.tq_join_put_probe(h, (L.TQColumn * 2)(*[c.tq() for c in p]), None, L.TQ_MEM_HOST))
    L.check(lib.tq_join_probe_eof(h))
    out = [Column.empty(INT64, 100) for _ in range(3)]
    from tinysql_b200.chunk import tq_array
    n, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_join_next(h, 100, tq_array(out, 100), C.byref(n), C.byref(eof)))
    assert n.value == 64 and out[0].values[:64].tolist() == [0] * 64 and out[2].values[:64].tolist() == list(range(64))
    L.check(lib.tq_join_destroy(h))
    # a negative key count is still refused
    bta = (C.c_int32 * 1)(INT64)
    d = L.TQJoinDesc(INNER_JOIN, 0, 1, bta, 1, bta, -1, None, None, 0, 0)
    hh = C.c_void_p()
    assert lib.tq_join_create(C.byref(d), C.byref(hh)) == L.TQ_ERR_INVALID_ARG
