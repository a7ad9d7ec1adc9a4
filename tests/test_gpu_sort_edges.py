"""GPU edge tests of SortExec / TopNExec / MergeJoinExec (csrc/sort.cu) against the exact reference of tests/sort_ref.py.

Every family of sort_ref runs through the operators twice: from host chunks, and (FLOAT columns excepted: they enter from
host memory only) from device columns put in ragged pieces.  Results are compared in order with the reference; a row-id
payload column makes the order of ties visible.  Each sort's digit-pass count (tq_sort_stats) must equal the restatement, so
the skip mask is pinned in both directions.  The merge join also runs a 2^26-row result (4096 groups of 16384 inner rows)
checked row by row, and the two result sizes past 2^32 rows that must be refused: one whose emit counts add up past 2^32
inside a single 4096-row tile of the scan, one that only does so across tiles.  The bodies also run under the CPU emulation
(test_emu_sort_edges.py)."""
import ctypes as C

import numpy as np
import pytest

import sort_ref as R
import test_gpu_zz_device_varlen as TV
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import INT64, Column
from tinysql_b200.executor import MergeJoinExec, MockDataSource, SortExec, TopNExec

pytestmark = pytest.mark.gpu

SORTS = R.sort_families(np.random.default_rng(7))
MJS = R.mj_keys(np.random.default_rng(8)) + R.mj_unsorted()
JOINS = [(R.INNER, False), (R.LEFT, False), (R.RIGHT, True)]
NE = 5                                             # TQ_CMP_NE


def sort_stats(lib, h):
    st = (C.c_int64 * 4)()
    L.check(lib.tq_sort_stats(h, st))
    return st[3]


def sort_host(lib, case, by, off, cnt, chunk):
    src = MockDataSource(case.types, case.columns(), chunk)
    e = SortExec(src, by) if off == 0 and cnt < 0 else TopNExec(src, by, off, cnt)
    e.Open()
    got = e.drain()
    passes = sort_stats(lib, e.handle)
    e.Close()
    return got.rows(), passes


def sort_device(lib, case, by, off, cnt, bounds):
    types = case.types
    d = L.TQSortDesc(len(types), TV.i32(types), len(by), TV.i32([c for c, _ in by]), TV.i32([1 if x else 0 for _, x in by]), off, cnt)
    h = C.c_void_p()
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    for dcs, arr in TV.device_pieces(case.columns(), bounds):
        L.check(lib.tq_sort_put(h, arr, L.TQ_MEM_DEVICE))
        TV.scribble_cells(lib, dcs)
        TV.free_all(dcs)
    L.check(lib.tq_sort_eof(h))
    out = (L.TQColumn * len(types))()
    n, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_sort_next_device(h, out, C.byref(n), C.byref(eof)))
    got = TV.lent_to_host(types, out, n.value).rows() if n.value else []
    passes = sort_stats(lib, h)
    L.check(lib.tq_sort_destroy(h))
    return got, passes


def sort_family_body(lib, case):
    R.check_family([case])
    rng = np.random.default_rng(len(case.name))
    for by, off, cnt in case.sorts:
        want = R.canon_rows(R.sort_rows(case.rows(), by, off, cnt))
        want_passes = R.passes(case.types, case.cols, case.nullable, by, off, cnt)
        for chunk in (1024, 77):
            got, passes = sort_host(lib, case, by, off, cnt, chunk)
            assert R.canon_rows(got) == want, (case.name, by, off, cnt, chunk)
            assert passes == want_passes, (case.name, by, off, cnt, chunk)
        if not case.has_float32():
            got, passes = sort_device(lib, case, by, off, cnt, TV.ragged_bounds(rng, case.n, max(case.n // 3, 1), 1))
            assert R.canon_rows(got) == want, (case.name, by, off, cnt, "device")
            assert passes == want_passes, (case.name, by, off, cnt, "device")


def too_many_by_items_body(lib):
    by = R.TOO_MANY_BY
    d = L.TQSortDesc(1, TV.i32([INT64]), len(by), TV.i32([c for c, _ in by]), TV.i32([0] * len(by)), 0, -1)
    h = C.c_void_p()
    assert lib.tq_sort_create(C.byref(d), C.byref(h)) == L.TQ_ERR_INVALID_ARG
    d = L.TQSortDesc(1, TV.i32([INT64]), R.SORT_MAX_BY, TV.i32([0] * R.SORT_MAX_BY), TV.i32([0] * R.SORT_MAX_BY), 0, -1)
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    L.check(lib.tq_sort_destroy(h))


def mj_host(case, jt, oir, sel=None, default_inner=None, conds=(), chunk=1024):
    flt = None
    if sel is not None:
        sel = np.asarray(sel, dtype=np.uint8)
        pos = [0]

        def flt(chk):
            lo = pos[0]
            pos[0] += chk.num_rows()
            return sel[lo: pos[0]]
    e = MergeJoinExec(MockDataSource(case.otypes, case.ocolumns(), chunk), MockDataSource(case.types, case.columns(), chunk), case.ok, case.ik, jt, oir, flt,
                      default_inner=default_inner, other_conditions=conds)
    e.Open()
    try:
        return e.drain().rows()
    finally:
        e.Close()


def mj_device(lib, case, jt, oir, rng):
    got = TV.mjoin_device(lib, jt, oir, case.types, case.columns(), case.otypes, case.ocolumns(), case.ik, case.ok,
                          TV.ragged_bounds(rng, case.n, max(case.n // 3, 1), 1), TV.ragged_bounds(rng, len(case.ocols[0]), max(len(case.ocols[0]) // 4, 1), 1))
    return got.rows() if got.num_rows() else []


def mj_family_body(lib, case):
    R.check_family([case])
    rng = np.random.default_rng(len(case.name))
    if case.refused:
        for run in (lambda: mj_host(case, R.INNER, False), lambda: mj_device(lib, case, R.INNER, False, rng)):
            with pytest.raises(L.TQError) as ei:
                run()
            assert ei.value.status == L.TQ_ERR_STATE, case.name
        return
    no = len(case.ocols[0])
    sel = [int(i % 3 != 1) for i in range(no)]
    dflt = [None] * (len(case.types) - 1) + [-7]        # defaultInner of the inner row id
    for jt, oir in JOINS:
        assert R.canon_rows(mj_host(case, jt, oir)) == R.canon_rows(R.mj_expect(case, jt, oir)), (case.name, jt, oir)
        assert R.canon_rows(mj_host(case, jt, oir, sel, chunk=50)) == R.canon_rows(R.mj_expect(case, jt, oir, sel)), (case.name, jt, oir, "sel")
        if not case.has_float32():
            assert R.canon_rows(mj_device(lib, case, jt, oir, rng)) == R.canon_rows(R.mj_expect(case, jt, oir)), (case.name, jt, oir, "device")
    got = mj_host(case, R.LEFT, False, sel, default_inner=dflt)
    assert R.canon_rows(got) == R.canon_rows(R.mj_expect(case, R.LEFT, False, sel, dflt)), (case.name, "defaultInner")


def size_guard_body(shape, with_conds):
    """every outer row and every inner row has the key 0: the result would have outer x inner > 2^32 rows, which the finish
    refuses before it sizes anything by that total"""
    no, ni = R.GUARD_SHAPES[shape]
    icols, ocols = [Column(INT64, np.zeros(ni, np.int64))], [Column(INT64, np.zeros(no, np.int64))]
    conds = [(NE, 0, None, INT64, 7)] if with_conds else ()          # outer key != 7: true for every pair
    e = MergeJoinExec(MockDataSource([INT64], ocols, 1 << 16), MockDataSource([INT64], icols, 1 << 16), [0], [0], R.INNER, False, other_conditions=conds)
    e.Open()
    try:
        with pytest.raises(L.TQError) as ei:
            e.drain()
    finally:
        e.Close()
    assert ei.value.status == L.TQ_ERR_INVALID_ARG, shape
    assert "exceeds 2^32" in str(ei.value)


@pytest.mark.parametrize("case", SORTS, ids=[c.name for c in SORTS])
def test_sort_family(lib, case):
    sort_family_body(lib, case)


def test_sort_refuses_more_than_eight_by_items(lib):
    too_many_by_items_body(lib)


@pytest.mark.parametrize("case", MJS, ids=[c.name for c in MJS])
def test_merge_join_family(lib, case):
    mj_family_body(lib, case)


def test_merge_join_big_groups(lib):
    """4096 outer rows, each the key of one group of 16384 inner rows: result row t joins outer row t // 16384 with the
    inner row t % 16384 of its group.  Device puts, result lent from the device and checked column by column."""
    no, g = R.BIG_GROUPS
    ni = no * g
    outer = [Column(INT64, np.arange(no, dtype=np.int64))]
    inner = [Column(INT64, np.repeat(np.arange(no, dtype=np.int64), g)), Column(INT64, np.tile(np.arange(g, dtype=np.int64), no))]
    md = L.TQMJoinDesc(R.INNER, 0, 2, TV.i32([INT64, INT64]), 1, TV.i32([INT64]), 1, TV.i32([0]), TV.i32([0]), None, None)
    h = C.c_void_p()
    L.check(lib.tq_mjoin_create(C.byref(md), C.byref(h)))
    for side, cols, put in ((0, inner, lib.tq_mjoin_put_inner), (1, outer, lib.tq_mjoin_put_outer)):
        for dcs, arr in TV.device_pieces(cols, [0, len(cols[0].values) // 3, len(cols[0].values)]):
            L.check(put(h, arr, L.TQ_MEM_DEVICE) if side == 0 else put(h, arr, None, L.TQ_MEM_DEVICE))
            TV.free_all(dcs)
    del inner
    L.check(lib.tq_mjoin_finish(h))
    out = (L.TQColumn * 3)()
    n, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_mjoin_next_device(h, out, C.byref(n), C.byref(eof)))
    assert n.value == ni
    t = np.arange(ni, dtype=np.int64)
    for c, want in ((0, t // g), (1, t // g), (2, t % g)):     # outer key, inner key, inner position in its group
        got = np.empty(ni, dtype=np.int64)
        L.check(lib.tq_memcpy_d2h(got.ctypes.data, out[c].data, got.nbytes))
        assert np.array_equal(got, want), c
        del got
    L.check(lib.tq_mjoin_destroy(h))


@pytest.mark.parametrize("shape", ["i", "ii"])
@pytest.mark.parametrize("with_conds", [False, True])
def test_merge_join_result_past_2_32_rows_is_refused(lib, shape, with_conds):
    assert R.guard_total(shape) > 1 << 32 and R.guard_wraps_one_tile(shape) == (shape == "i")
    size_guard_body(shape, with_conds)
