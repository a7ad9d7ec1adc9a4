"""GPU parity for OtherConditions as an expression program inside the hash join and the merge join
(tq_join_set_other_program / tq_mjoin_set_other_program) against the restatement of tryToMatchInners -> filter -> onMissMatch
in join_program_oracle.py: the joined rows, the miss rows of outer joins, the division-by-zero warnings, the error status, and
which rows can raise at all (only key-matched rows in VecEvalBool's evaluation set)."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O
from join_program_oracle import OracleError, conds_to_program, join_with_program
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, FLOAT32, FLOAT64, INT64, UINT64, Column, DeviceColumn, device_to_host
from tinysql_b200.executor import INNER_JOIN, LEFT_OUTER_JOIN, RIGHT_OUTER_JOIN, HashJoinExec, MergeJoinExec, MockDataSource
from tinysql_b200.expression import Col, Const, Func, JoinProgram
from util import assert_same_multiset, assert_same_ordered, gen_col

pytestmark = pytest.mark.gpu

TP = {INT64: "int", UINT64: "uint", FLOAT64: "real"}
JOINS = [(INNER_JOIN, False), (INNER_JOIN, True), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)]


def _flt(sel):
    """the outer filter's result for each chunk the executor fetches, from one selection vector"""
    if sel is None:
        return None
    sel = np.asarray(sel, dtype=np.uint8)
    pos = [0]

    def f(chk):
        lo = pos[0]
        pos[0] += chk.num_rows()
        return sel[lo: pos[0]]
    return f


def run(kind, jt, oir, it, ic, ot, oc, ik, ok, program=(), conds=(), sel=None, batch=0, default_inner=None, chunk=1 << 16):
    """-> (rows, division-by-zero warnings) of HashJoinExec (kind 'hash') or MergeJoinExec ('merge')"""
    outer, inner = MockDataSource(ot, oc, chunk), MockDataSource(it, ic, chunk)
    if kind == "hash":
        e = HashJoinExec(outer, inner, ok, ik, jt, oir, _flt(sel), batch, other_program=program, other_conditions=conds, default_inner=default_inner)
    else:
        e = MergeJoinExec(outer, inner, ok, ik, jt, oir, _flt(sel), default_inner=default_inner, other_conditions=conds, other_program=program)
    e.Open()
    try:
        return e.drain(), e.warnings
    finally:
        e.Close()


class Tables:
    """inner (build) and outer (probe) tables with named columns; col(name) is that column of the joined row left ++ right"""

    def __init__(self, oir, inner, outer):
        self.oir = oir
        self.inames, self.onames = list(inner), list(outer)
        self.ic, self.oc = list(inner.values()), list(outer.values())
        self.it, self.ot = [c.tp for c in self.ic], [c.tp for c in self.oc]
        names = (self.inames + self.onames) if oir else (self.onames + self.inames)
        self.pos = {n: i for i, n in enumerate(names)}
        self.types = (self.it + self.ot) if oir else (self.ot + self.it)

    def col(self, name):
        return Col(self.pos[name], TP[self.types[self.pos[name]]])


def make_tables(rng, oir, ni, no, sort=False):
    ndv = max(ni // 3, 2)
    ik, ok = gen_col(rng, INT64, ni, 0.05, 0, ndv), gen_col(rng, INT64, no, 0.05, 0, ndv + 2)
    if sort:   # the merge join's children are sorted by the key (NULLs first, as the planner's sort leaves them)
        ik = Column(INT64, np.sort(np.where(ik.not_null(), ik.values, -1)), np.sort(np.where(ik.not_null(), ik.values, -1)) >= 0)
        ok = Column(INT64, np.sort(np.where(ok.not_null(), ok.values, -1)), np.sort(np.where(ok.not_null(), ok.values, -1)) >= 0)
    inner = {"ik": ik, "iid": Column(INT64, np.arange(ni)), "iv": gen_col(rng, INT64, ni, 0.1), "is": gen_col(rng, INT64, ni, 0.1, -50, 50),
             "iu": gen_col(rng, UINT64, ni, 0.1, 0, 50), "id": Column(FLOAT64, rng.integers(-2, 3, ni) * 0.5, rng.random(ni) > 0.1),
             "if32": Column(FLOAT32, rng.random(ni).astype(np.float32), rng.random(ni) > 0.1),
             "istr": Column(BYTES, [b"s%d" % v if v else None for v in rng.integers(0, 50, ni)])}
    outer = {"od": Column(FLOAT64, rng.integers(-3, 4, no) * 1.0, rng.random(no) > 0.1), "ok": ok, "ov": gen_col(rng, INT64, no, 0.1, -50, 50),
             "oid": Column(INT64, np.arange(no)), "ou": gen_col(rng, UINT64, no, 0.1, 0, 60)}
    return Tables(oir, inner, outer)


def programs(t):
    c = t.col
    return [
        [Func("gt", Func("plus", c("iv"), c("ov")), Const(10))],                                            # BIGINT + near +-2^62
        [Func("or", Func("lt", Func("minus", c("ov"), c("iv")), Const(0)), Func("isnull", c("ov"))),
         Func("not", Func("eq", c("iu"), Const(3, "uint")))],                                               # OR, IS NULL, NOT
        [Func("ge", Func("if", Func("gt", c("ov"), Const(0)), c("ov"), Func("mul", c("ov"), Const(-2))), Func("ifnull", c("is"), Const(0)))],
        [Func("in", c("ov"), c("is"), Const(3), Const(None))],                                               # IN with a NULL constant
        [Func("gt", Func("div", c("od"), c("id")), Const(0.5, "real"))],                                     # real division by zero
        [Func("lt", Func("plus", c("iu"), Const(5, "uint")), c("ou")), Func("ne", c("is"), c("ov"))],        # BIGINT UNSIGNED
        [Func("or", Func("eq", c("ov"), Const(None)), Func("gt", Func("mul", c("is"), c("ov")), Const(-100)))],
    ]


def check(kind, t, program, jt, sel=None, batch=0, default_inner=None, ik=("ik",), ok=("ok",), ordered=False):
    iks = [t.inames.index(n) for n in ik]
    oks = [t.onames.index(n) for n in ok]
    try:
        want, wwarn = join_with_program(kind, jt, t.oir, t.it, t.ic, t.ot, t.oc, iks, oks, program, sel, default_inner)
    except OracleError as oe:
        with pytest.raises(L.TQError) as ei:
            run(kind, jt, t.oir, t.it, t.ic, t.ot, t.oc, iks, oks, program, sel=sel, batch=batch, default_inner=default_inner)
        assert ei.value.status == oe.status
        return None, None
    got, warn = run(kind, jt, t.oir, t.it, t.ic, t.ot, t.oc, iks, oks, program, sel=sel, batch=batch, default_inner=default_inner)
    (assert_same_ordered if ordered else assert_same_multiset)(got, want)
    assert warn == wwarn
    return got, warn


def assert_probe_then_build_order(got, t):
    """the one-table path's order: probe row ascending, build insertion ascending inside a probe row"""
    pid, bid = got.cols[t.pos["oid"]].values, got.cols[t.pos["iid"]].values
    assert np.all(np.diff(pid) >= 0)
    same = np.diff(pid) == 0
    assert np.all(np.diff(bid)[same] > 0)


@pytest.mark.parametrize("jt,oir", JOINS)
@pytest.mark.parametrize("ni,no", [(300, 5000), (270000, 300000)])
def test_hash_join_program_vs_oracle(lib, jt, oir, ni, no):
    """the one-table path (build side below 2^18 rows, checked in order: every program) and the partitioned path (three
    programs); duplicate and NULL keys, NULL payloads, FLOAT and var-len payloads the program does not read"""
    rng = np.random.default_rng(ni + jt * 7 + int(oir))
    t = make_tables(rng, oir, ni, no)
    for i, prog in enumerate(programs(t)):
        if ni >= (1 << 18) and i not in (0, 1, 4):
            continue
        got, warn = check("hash", t, prog, jt)
        assert got is not None
        if ni < (1 << 18):
            assert_probe_then_build_order(got, t)
        if i == 4:
            assert warn > 0   # the division program counts warnings


@pytest.mark.parametrize("jt,oir", JOINS)
def test_hash_join_program_batches_filter_defaults_multikey(lib, jt, oir):
    """small probe batches (batch boundaries inside the probe side), the outer filter, defaultInner, a two-column key"""
    rng = np.random.default_rng(31 + jt + int(oir))
    t = make_tables(rng, oir, 2000, 20000)
    sel = (rng.random(20000) > 0.25).astype(np.uint8)
    dflt = [None, -1, 7, None, 5, 2.5, None, None] if jt != INNER_JOIN else None
    for prog in programs(t)[:3] + programs(t)[4:5]:
        assert check("hash", t, prog, jt, sel=sel, batch=1000, default_inner=dflt)[0] is not None
    assert check("hash", t, programs(t)[0], jt, sel=sel, batch=1000, ik=("ik", "is"), ok=("ok", "ov"))[0] is not None


def test_hash_join_program_device_input(lib):
    """device columns in (TQ_MEM_DEVICE), the filtered batches lent by tq_join_next_device"""
    rng = np.random.default_rng(17)
    nb, npr = 50000, 400000
    bcols = [Column(INT64, rng.integers(0, nb // 2, nb)), gen_col(rng, INT64, nb, 0.1, -100, 100), Column(FLOAT64, rng.integers(-2, 3, nb) * 0.5)]
    pcols = [Column(INT64, rng.integers(0, nb // 2, npr)), gen_col(rng, INT64, npr, 0.1, -100, 100), Column(FLOAT64, rng.integers(-9, 9, npr) * 1.5)]
    bt, pt = [c.tp for c in bcols], [c.tp for c in pcols]
    # output = b0 b1 b2 p0 p1 p2 (outer_is_right): b1 * p1 > 0 and p2 / b2 < 10
    prog = [Func("gt", Func("mul", Col(1), Col(4)), Const(0)), Func("lt", Func("div", Col(5, "real"), Col(2, "real")), Const(10.0, "real"))]
    want, wwarn = join_with_program("hash", INNER_JOIN, True, bt, bcols, pt, pcols, [0], [0], prog)
    d_b = [DeviceColumn.from_host(c) for c in bcols]
    d_p = [DeviceColumn.from_host(c) for c in pcols]
    ta, tb, kk = (C.c_int32 * 3)(*bt), (C.c_int32 * 3)(*pt), (C.c_int32 * 1)(0)
    d = L.TQJoinDesc(INNER_JOIN, 1, 3, ta, 3, tb, 1, kk, kk, 0, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    try:
        JoinProgram(prog).set_on(lib.tq_join_set_other_program, h)
        L.check(lib.tq_join_put_build(h, (L.TQColumn * 3)(*[c.tq() for c in d_b]), L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        L.check(lib.tq_join_put_probe(h, (L.TQColumn * 3)(*[c.tq() for c in d_p]), None, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_probe_eof(h))
        parts = [[] for _ in range(6)]
        while True:
            out, n, eof = (L.TQColumn * 6)(), C.c_int64(0), C.c_int32(0)
            L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
            if n.value == 0 and eof.value:
                break
            for c, tp in enumerate(bt + pt):
                parts[c].append(device_to_host(tp, out[c].data, out[c].null_bitmap, n.value))
        w = C.c_int64(0)
        L.check(lib.tq_join_warnings(h, C.byref(w)))
    finally:
        lib.tq_join_destroy(h)
        for c in d_b + d_p:
            c.free()
    from tinysql_b200.chunk import Chunk
    got = Chunk([Column(tp, np.concatenate([p.values for p in ps]), np.concatenate([p.not_null() for p in ps])) for tp, ps in zip(bt + pt, parts)])
    assert_same_multiset(got, want)
    assert w.value == wwarn


@pytest.mark.parametrize("jt,oir", JOINS)
def test_merge_join_program_vs_oracle(lib, jt, oir, ni=20000, no=30000):
    """in the reference's order; NULL keys, the outer filter, defaultInner, FLOAT and var-len payloads"""
    rng = np.random.default_rng(70 + jt + 3 * int(oir))
    t = make_tables(rng, oir, ni, no, sort=True)
    sel = (rng.random(no) > 0.1).astype(np.uint8)
    dflt = [None, -1, 7, None, 5, 2.5, None, None] if jt != INNER_JOIN else None
    for prog in programs(t):
        assert check("merge", t, prog, jt, sel=sel, default_inner=dflt, ordered=True)[0] is not None


def _edge_tables(oir, tp, flag=(1, 1, 1, 1), key_nn=(True, True, True, True)):
    """outer row 1 (key 2) meets inner row 1 (key 2) and both carry a value whose sum overflows tp; outer row 3 carries one too,
    but its key 4 has no inner match.  Both children are sorted by the key, as the merge join needs."""
    big = (1 << 62) if tp == INT64 else (1 << 63)
    inner = {"ik": Column(INT64, [1, 2, 3, 5]), "iv": Column(tp, [1, big, 1, big])}
    outer = {"ok": Column(INT64, [1, 2, 3, 4], list(key_nn)), "ov": Column(tp, [1, big, 1, big]), "flag": Column(INT64, list(flag)),
             "oid": Column(INT64, [0, 1, 2, 3])}
    return Tables(oir, inner, outer)


@pytest.mark.parametrize("kind", ["hash", "merge"])
@pytest.mark.parametrize("jt,oir", [(INNER_JOIN, False), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)])
def test_overflow_raises_only_for_evaluated_rows(lib, kind, jt, oir):
    for tp, status in ((INT64, L.TQ_ERR_OVERFLOW_BIGINT), (UINT64, L.TQ_ERR_OVERFLOW_BIGINT_UNSIGNED)):
        zero = Const(0, TP[tp])
        t = _edge_tables(oir, tp)
        ovf = Func("gt", Func("plus", t.col("iv"), t.col("ov")), zero)
        # in the evaluation set: big + big on the joined row of outer row 1
        with pytest.raises(L.TQError) as ei:
            run(kind, jt, oir, t.it, t.ic, t.ot, t.oc, [0], [0], [ovf])
        assert ei.value.status == status
        assert check(kind, t, [ovf], jt)[0] is None
        # the same row dropped by an earlier FILTER item
        t = _edge_tables(oir, tp, flag=(1, 0, 1, 1))
        assert check(kind, t, [Func("ne", t.col("flag"), Const(0)), ovf], jt)[0] is not None
        # outside the outer filter (selected == 0)
        assert check(kind, t, [ovf], jt, sel=[1, 0, 1, 1])[0] is not None
        # ov + ov overflows on outer rows 1 and 3: row 1 has a NULL key, row 3 no key match
        t = _edge_tables(oir, tp, key_nn=(True, False, True, True))
        if kind == "merge":   # the merge join's outer child is sorted with its NULL keys first
            t.oc = [Column(c.tp, c.values[[1, 0, 2, 3]], c.not_null()[[1, 0, 2, 3]]) for c in t.oc]
        assert check(kind, t, [Func("gt", Func("plus", t.col("ov"), t.col("ov")), zero)], jt)[0] is not None
    # DOUBLE: a product out of range
    t = Tables(oir, {"ik": Column(INT64, [1, 2]), "iv": Column(FLOAT64, [1.0, 1e300])}, {"ok": Column(INT64, [1, 2]), "ov": Column(FLOAT64, [1e300, 1e300])})
    with pytest.raises(L.TQError) as ei:
        run(kind, jt, oir, t.it, t.ic, t.ot, t.oc, [0], [0], [Func("gt", Func("mul", t.col("iv"), t.col("ov")), Const(0.0, "real"))])
    assert ei.value.status == L.TQ_ERR_OVERFLOW_DOUBLE


def _ops(prog):
    return (L.TQExprOp * max(len(prog), 1))(*prog)


def _set(setter, h, cols, ops):
    return setter(h, len(cols), (C.c_int32 * max(len(cols), 1))(*cols), len(ops), _ops(ops))


@pytest.mark.parametrize("kind", ["hash", "merge"])
def test_abi_rejections(lib, kind):
    """malformed programs and wrong column types are refused before any device work; one form per handle"""
    types = [INT64, INT64, FLOAT32, BYTES]   # output = outer ++ inner = 4 + 4 columns: 2, 3, 6, 7 are FLOAT / var-len
    ta, kk = (C.c_int32 * 4)(*types), (C.c_int32 * 1)(0)
    X = L.TQExprOp
    cmp = X(1, 0, 0, 1, 0, 0, 0, 0, 0)         # CMP_INT LT r0 r1
    flt = X(9, 0, 2, 0, 0, 0, 0, 0, 0)         # FILTER r2

    def handle():
        h = C.c_void_p()
        if kind == "hash":
            L.check(lib.tq_join_create(C.byref(L.TQJoinDesc(LEFT_OUTER_JOIN, 0, 4, ta, 4, ta, 1, kk, kk, 0, 0)), C.byref(h)))
        else:
            L.check(lib.tq_mjoin_create(C.byref(L.TQMJoinDesc(LEFT_OUTER_JOIN, 0, 4, ta, 4, ta, 1, kk, kk, None, None)), C.byref(h)))
        return h
    set_prog = lib.tq_join_set_other_program if kind == "hash" else lib.tq_mjoin_set_other_program
    set_conds = lib.tq_join_set_other_conditions if kind == "hash" else lib.tq_mjoin_set_other_conditions
    destroy = lib.tq_join_destroy if kind == "hash" else lib.tq_mjoin_destroy
    cases = [
        ([0, 4], [X(1, 0, 0, 5, 0, 0, 0, 0, 0), flt], L.TQ_ERR_INVALID_ARG),      # reads a register before it is written
        ([0, 4], [cmp, X(10, 0, 0, 0, 0, 0, 0, 0, 0), flt], L.TQ_ERR_INVALID_ARG),  # COMPACT
        ([0, 4], [cmp], L.TQ_ERR_INVALID_ARG),                                      # no FILTER
        ([0, 1, 4, 5, 0, 1, 4, 5, 0], [cmp, flt], L.TQ_ERR_INVALID_ARG),            # 9 inputs
        ([0, 4], [cmp] * 32 + [flt], L.TQ_ERR_INVALID_ARG),                         # 33 ops
        ([0, 9], [cmp, flt], L.TQ_ERR_INVALID_ARG),                                 # no such column
        ([0, 2], [cmp, flt], L.TQ_ERR_UNSUPPORTED_TYPE),                            # FLOAT input
        ([7, 4], [cmp, flt], L.TQ_ERR_UNSUPPORTED_TYPE),                            # var-len input
    ]
    for cols, ops, status in cases:
        h = handle()
        assert _set(set_prog, h, cols, ops) == status, (cols, status)
        assert _set(set_prog, h, [0, 4], [cmp, flt]) == L.TQ_OK      # a refused call leaves the handle as it was
        destroy(h)
    conds = (L.TQJoinCond * 1)(L.TQJoinCond(0, 0, 4, 0, 0))
    h = handle()
    assert _set(set_prog, h, [0, 4], [cmp, flt]) == L.TQ_OK
    assert set_conds(h, 1, conds) == L.TQ_ERR_STATE
    assert _set(set_prog, h, [0, 4], [cmp, flt]) == L.TQ_ERR_STATE
    destroy(h)
    h = handle()
    assert set_conds(h, 1, conds) == L.TQ_OK
    assert _set(set_prog, h, [0, 4], [cmp, flt]) == L.TQ_ERR_STATE
    destroy(h)


@pytest.mark.parametrize("jt,oir", JOINS)
def test_program_form_equals_comparison_form(lib, jt, oir):
    """the same conditions given as tq_join_cond comparisons and as a program: identical results on the device"""
    rng = np.random.default_rng(5 + jt + int(oir))
    for kind, (ni, no) in (("hash", (270000, 300000)), ("hash", (3000, 20000)), ("merge", (20000, 30000))):
        t = make_tables(rng, oir, ni, no, sort=kind == "merge")
        p = t.pos
        for conds in ([(0, p["is"], p["ov"])], [(3, p["id"], p["od"]), (5, p["iu"], None, UINT64, 7), (1, p["iv"], None, INT64, 0)]):
            a, _ = run(kind, jt, oir, t.it, t.ic, t.ot, t.oc, [0], [1], conds=conds)
            b, wb = run(kind, jt, oir, t.it, t.ic, t.ot, t.oc, [0], [1], conds_to_program(conds, t.types))
            (assert_same_ordered if kind == "merge" else assert_same_multiset)(a, b)
            assert wb == 0
            if kind == "hash":
                assert_same_multiset(a, O.hash_join(jt, oir, t.it, t.ic, t.ot, t.oc, [0], [1], None, conds))
