"""GPU: the fixed-width builtins at their overflow and sign boundaries in every kernel that runs them — k_map / k_in_int /
k_filter_int behind tq_vec_*, k_expr_prog behind tq_expr_eval, k_oc_eval behind the hash join's program and k_mj_prog behind
the merge join's — against the restatement of the reference's per-row statements (vec_statements.py) and the oracle.

Values: every pool row the restatement lets through, in one call, bit-exact, with NULL rows whose slots hold raising operands.
Errors: one sample row per branch tag of each op and sign mix, alone among non-raising rows at the start, both sides of the
first 64-row group boundary, the last row and (host input) past the first 4M-row slab; each call returns the restatement's
kind, and the same rows raise nothing when an operand is NULL or a filter removed the row first.  Error order: when several
ops raise different kinds, the first op in evaluation order decides."""
import ctypes as C
from functools import lru_cache

import numpy as np
import pytest

import edge_operands as EO
import oracle_py as O
import test_gpu_join_program as TJ
import vec_statements as V
from test_gpu_expr_program import OracleError, check, oracle_select_project
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import FLOAT64, INT64, UINT64, Column, DeviceColumn
from tinysql_b200.executor import INNER_JOIN, LEFT_OUTER_JOIN
from tinysql_b200.expression import Col, Const, ExprProgram, Func

pytestmark = pytest.mark.gpu

HOST, DEVICE = L.TQ_MEM_HOST, L.TQ_MEM_DEVICE
SLAB_ROWS = 1 << 22            # expr.cu: rows per host-path slab
ARITH_NAMES = ["plus", "minus", "mul", "div"]


def _tp(unsigned):
    return UINT64 if unsigned else INT64


def _et(tp):
    return {INT64: "int", UINT64: "uint", FLOAT64: "real"}[tp]


# ------------------------------------------------------------------ the raising ops: (kind, op, a unsigned, b unsigned)
class Spec:
    def __init__(self, kind, op=0, ua=False, ub=False):
        self.kind, self.op, self.ua, self.ub = kind, op, ua, ub
        self.ta = FLOAT64 if kind == "real" else _tp(ua)
        self.tb = FLOAT64 if kind == "real" else _tp(ub)
        self.out_tp = FLOAT64 if kind == "real" else (INT64 if kind == "neg" else _tp(ua or ub))

    def __repr__(self):
        if self.kind == "neg":
            return "neg_" + ("U" if self.ua else "S")
        if self.kind == "real":
            return ARITH_NAMES[self.op] + "_real"
        return ARITH_NAMES[self.op] + "_" + ("U" if self.ua else "S") + ("U" if self.ub else "S")

    def stmt(self, x, y):
        if self.kind == "int":
            return V.arith_int(self.op, x, y, self.ua, self.ub)
        if self.kind == "real":
            return V.arith_real(self.op, x, y)
        return V.neg_int(x, self.ua)

    def expr(self, a, b):
        """the op over Expr operands"""
        return Func("neg", a) if self.kind == "neg" else Func(ARITH_NAMES[self.op], a, b)

    def raising_tags(self):
        """every branch of the restatement that returns an error for this op and mix"""
        if self.kind == "neg":
            return {"UnaryMinusInt:229" if self.ua else "UnaryMinusInt:236"}
        if self.kind == "real":
            return [{"PlusReal:296 x>0", "PlusReal:296 x<0"}, {"MinusReal:83 x>0", "MinusReal:83 x<0"}, {"MultiplyReal:51"},
                    {"DivideReal:378"}][self.op]
        mix = ("U" if self.ua else "S") + ("U" if self.ub else "S")
        if self.op == 2:
            return {"MultiplyIntUnsigned:526"} if (self.ua or self.ub) else {"MultiplyInt:333"}
        return {("plus", "UU"): {"plusUU:435"}, ("plus", "US"): {"plusUS:451", "plusUS:454"}, ("plus", "SU"): {"plusSU:470", "plusSU:473"},
                ("plus", "SS"): {"plusSS:488 lh>0", "plusSS:488 lh<0"}, ("minus", "UU"): {"minusUU:212"},
                ("minus", "US"): {"minusUS:228", "minusUS:231"}, ("minus", "SU"): {"minusSU:247"},
                ("minus", "SS"): {"minusSS:262 lh>0", "minusSS:262 lh<0"}}[(ARITH_NAMES[self.op], mix)]


SPECS = ([Spec("int", op, ua, ub) for op in range(3) for ua, ub in EO.INT_MIXES] + [Spec("real", op) for op in range(4)]
         + [Spec("neg", 0, ua) for ua in (False, True)])


@lru_cache(maxsize=None)
def rows_of(spec):
    """-> (xs, ys, [(value, kind, tag)]) over the spec's edge pairs"""
    if spec.kind == "int":
        pairs = EO.int_pairs(spec.op, spec.ua, spec.ub)
    elif spec.kind == "real":
        pairs = EO.real_pairs(spec.op)
    else:
        pairs = sorted({(x, 0) for x in EO.pool(spec.ua)} | {(p[0], 0) for p in EO.int_pairs(0, spec.ua, spec.ua)[::5]})
    res = [spec.stmt(x, y) for x, y in pairs]
    return [p[0] for p in pairs], [p[1] for p in pairs], res


def samples(spec):
    """one raising row per branch tag (the first in pool order) -> [(x, y, kind, tag)]; asserts that every tag is reached"""
    xs, ys, res = rows_of(spec)
    seen = {}
    for x, y, (_, kind, tag) in zip(xs, ys, res):
        if kind is not None and tag not in seen:
            seen[tag] = (x, y, kind, tag)
    assert set(seen) == spec.raising_tags(), (spec, set(seen))
    return list(seen.values())


def value_rows(spec, n_mod, seed=0):
    """(a, b, want, want_nn, warnings): all non-raising rows once, padded to n == n_mod (mod 64); 20 % NULL rows, whose slots
    hold raising operands"""
    xs, ys, res = rows_of(spec)
    ok = [i for i, r in enumerate(res) if r[1] is None]
    bad = [i for i, r in enumerate(res) if r[1] is not None]
    n = ((len(ok) + 63) // 64) * 64 + n_mod
    rng = np.random.default_rng(seed + n_mod)
    idx = np.array(ok + list(rng.choice(ok, n - len(ok))))
    na, nb = EO.null_mask(rng, n), EO.null_mask(rng, n)
    if spec.kind == "neg":
        nb[:] = True
    nulls = np.nonzero(~(na & nb))[0]
    idx[nulls] = np.array(bad)[np.arange(len(nulls)) % len(bad)]   # NULL rows carry raising operands
    x = [xs[i] for i in idx]
    y = [ys[i] for i in idx]
    nn = na & nb
    want_nn = nn.copy()
    want = np.zeros(n, dtype=np.uint64)
    warnings = 0
    for r, i in enumerate(idx):
        if not nn[r]:
            continue
        v, _, tag = res[i]
        if v is None:              # division by zero: NULL and a warning
            want_nn[r] = False
            warnings += 1
        elif spec.kind == "real":
            want[r] = np.float64(v).view(np.uint64)
        else:
            want[r] = v
    return EO.column(x, spec.ta, na), EO.column(y, spec.tb, nb), want, want_nn, warnings


def error_rows(spec, x, y, pos, n, seed=0):
    """n rows of non-raising operands with the raising pair (x, y) at row pos"""
    xs, ys, res = rows_of(spec)
    ok = np.array([i for i, r in enumerate(res) if r[1] is None])
    rng = np.random.default_rng(seed)
    pick = ok[rng.integers(0, len(ok), min(n, 4096))]
    a = np.resize(EO.np_values([xs[i] for i in pick], spec.ta), n)
    b = np.resize(EO.np_values([ys[i] for i in pick], spec.tb), n)
    a[pos], b[pos] = x, y
    return Column(spec.ta, a), Column(spec.tb, b)


def positions(n, mem, big_ok=True):
    pos = [0, 63, 64, n - 1]
    return [(p, n) for p in pos] + ([(SLAB_ROWS + 5, SLAB_ROWS + 65)] if (mem == HOST and big_ok) else [])


# ------------------------------------------------------------------ calls with host or device columns
class Mem:
    """TQColumns for one call: host columns as they are, or copies in HBM (outputs read back by fetch)"""

    def __init__(self, mem):
        self.mem, self.keep, self.dev = mem, [], []

    def inp(self, col):
        self.keep.append(col)
        if self.mem == HOST:
            return col.tq()
        d = DeviceColumn.from_host(col)
        self.dev.append(d)
        return d.tq()

    def out(self, tp, n):
        if self.mem == HOST:
            c = Column.empty(tp, n)
            self.keep.append(c)
            return c.tq(), (lambda: c)
        d = DeviceColumn(tp, n)
        self.dev.append(d)
        return d.tq(), (lambda: d.to_host(n))

    def sel(self, n):
        """a selection vector of n bytes -> (pointer, fetch)"""
        if self.mem == HOST:
            s = np.zeros(max(n, 1), dtype=np.uint8)
            self.keep.append(s)
            return s.ctypes.data, (lambda: s[:n].copy())
        d = DeviceColumn(UINT64, (n + 7) // 8, with_bitmap=False)
        self.dev.append(d)

        def fetch():
            s = np.zeros(max(n, 1), dtype=np.uint8)
            L.check(L.load().tq_memcpy_d2h(s.ctypes.data, d._data.value, n))
            return s[:n]
        return d._data.value, fetch

    def free(self):
        for d in self.dev:
            d.free()


def vec_call(lib, spec, a, b, mem):
    """-> (status, result Column, warnings) of the spec's tq_vec_* entry point"""
    m = Mem(mem)
    try:
        ta = m.inp(a)
        to, get = m.out(spec.out_tp, a.length)
        dz = C.c_int64(0)
        if spec.kind == "int":
            tb = m.inp(b)
            st = lib.tq_vec_arith_int(spec.op, a.length, C.byref(ta), int(spec.ua), C.byref(tb), int(spec.ub), C.byref(to), mem)
        elif spec.kind == "real":
            tb = m.inp(b)
            st = lib.tq_vec_arith_real(spec.op, a.length, C.byref(ta), C.byref(tb), C.byref(to), C.byref(dz), mem)
        else:
            st = lib.tq_vec_unary(2, a.length, C.byref(ta), int(spec.ua), C.byref(to), mem)
        return st, (get() if st == 0 else None), dz.value
    finally:
        m.free()


def oracle_call(spec, a, b):
    if spec.kind == "int":
        rc, out = O.vec_arith_int(spec.op, a, b)
        return rc, out, 0
    if spec.kind == "real":
        return O.vec_arith_real(spec.op, a, b)
    rc, out = O.vec_unary(2, a)
    return rc, out, 0


def assert_values(got, want, want_nn):
    assert np.array_equal(got.not_null(), want_nn), f"NULL masks differ at {np.nonzero(got.not_null() != want_nn)[0][:8]}"
    bad = np.nonzero(got.raw()[want_nn] != want[want_nn])[0]
    assert bad.size == 0, f"values differ at non-NULL rows {np.nonzero(want_nn)[0][bad[:8]]}"


# ------------------------------------------------------------------ tq_vec_* arithmetic
@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("spec", SPECS, ids=repr)
def test_vec_arith_values(lib, spec, mem):
    for n_mod in (1, 63):
        a, b, want, want_nn, warn = value_rows(spec, n_mod)
        st, got, dz = vec_call(lib, spec, a, b, mem)
        assert st == 0
        assert_values(got, want, want_nn)
        assert dz == warn
        rc, ref, odz = oracle_call(spec, a, b)
        assert rc == 0 and odz == warn
        assert_values(ref, want, want_nn)


@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("spec", SPECS, ids=repr)
def test_vec_arith_errors(lib, spec, mem):
    smp = samples(spec)
    for x, y, kind, tag in smp:
        for pos, n in positions(129, mem):
            a, b = error_rows(spec, x, y, pos, n)
            assert vec_call(lib, spec, a, b, mem)[0] == kind, (tag, pos)
    # every sampled row at once, each with one operand NULL: nothing raises
    n = 64 * len(smp) + 1
    a, b = error_rows(spec, smp[0][0], smp[0][1], 0, n)
    na, nb = np.ones(n, dtype=bool), np.ones(n, dtype=bool)
    for k, (x, y, _, _) in enumerate(smp):
        for j, r in enumerate((64 * k, 64 * k + 63)):
            a.values[r], b.values[r] = x, y
            (na if (j == 0 or spec.kind == "neg") else nb)[r] = False
    a, b = Column(spec.ta, a.values, na), Column(spec.tb, b.values, nb)
    assert vec_call(lib, spec, a, b, mem)[0] == 0


def test_lt_plus_int_edges(lib):
    """the fused (a < b, a + b) of signed BIGINT columns: plusSS's two branches and VecCompareII at every edge pair"""
    spec = Spec("int", 0, False, False)
    for mem in (HOST, DEVICE):
        for n_mod in (1, 63):
            a, b, want, want_nn, _ = value_rows(spec, n_mod)
            m = Mem(mem)
            try:
                ta, tb = m.inp(a), m.inp(b)
                tl, get_lt = m.out(INT64, a.length)
                tp, get_p = m.out(INT64, a.length)
                assert lib.tq_vec_lt_plus_int(a.length, C.byref(ta), C.byref(tb), C.byref(tl), C.byref(tp), mem) == 0
                lt, plus = get_lt(), get_p()
            finally:
                m.free()
            assert_values(plus, want, want_nn)
            wlt = np.array([V.cmp_result(0, V.compare_int(int(x), int(y), False, False)[0]) for x, y in zip(a.values, b.values)], dtype=np.uint64)
            assert_values(lt, wlt, want_nn)
        for x, y, kind, tag in samples(spec):
            for pos, n in positions(129, mem):
                a, b = error_rows(spec, x, y, pos, n)
                m = Mem(mem)
                try:
                    ta, tb = m.inp(a), m.inp(b)
                    tl, _ = m.out(INT64, n)
                    tp, _ = m.out(INT64, n)
                    assert lib.tq_vec_lt_plus_int(n, C.byref(ta), C.byref(tb), C.byref(tl), C.byref(tp), mem) == kind, (tag, pos)
                finally:
                    m.free()


# ------------------------------------------------------------------ comparisons, IN, toBool
def _cmp_pairs(ua, ub):
    return EO.int_pairs(0, ua, ub)[::3] + [(x, y) for x in EO.pool(ua) for y in EO.pool(ub)]


@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("ua,ub", EO.INT_MIXES)
def test_vec_compare_int_edges(lib, ua, ub, mem):
    pairs = _cmp_pairs(ua, ub)
    n = ((len(pairs) + 63) // 64) * 64 + 63
    pairs = (pairs * 2)[:n]
    rng = np.random.default_rng(3)
    a = EO.column([p[0] for p in pairs], _tp(ua), EO.null_mask(rng, n))
    b = EO.column([p[1] for p in pairs], _tp(ub), EO.null_mask(rng, n))
    nn = a.not_null() & b.not_null()
    for op in range(6):
        want = np.array([V.cmp_result(op, V.compare_int(x, y, ua, ub)[0]) for x, y in pairs], dtype=np.uint64)
        m = Mem(mem)
        try:
            ta, tb = m.inp(a), m.inp(b)
            to, get = m.out(INT64, n)
            assert lib.tq_vec_compare_int(op, n, C.byref(ta), int(ua), C.byref(tb), int(ub), C.byref(to), mem) == 0
            assert_values(get(), want, nn)
        finally:
            m.free()
        assert_values(O.vec_compare_int(op, a, b)[1], want, nn)


@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
def test_vec_compare_real_and_filters_edges(lib, mem):
    pool = EO.FLOAT64_FILTER_POOL
    pairs = [(x, y) for x in pool for y in pool]
    n = ((len(pairs) + 63) // 64) * 64 + 1
    pairs = (pairs * 2)[:n]
    rng = np.random.default_rng(4)
    a = EO.column([p[0] for p in pairs], FLOAT64, EO.null_mask(rng, n))
    b = EO.column([p[1] for p in pairs], FLOAT64, EO.null_mask(rng, n))
    nn = a.not_null() & b.not_null()
    for op in range(6):
        want = np.array([V.cmp_result(op, V.compare_float(x, y)) for x, y in pairs], dtype=np.uint64)
        m = Mem(mem)
        try:
            ta, tb = m.inp(a), m.inp(b)
            to, get = m.out(INT64, n)
            assert lib.tq_vec_compare_real(op, n, C.byref(ta), C.byref(tb), C.byref(to), mem) == 0
            assert_values(get(), want, nn)
        finally:
            m.free()
    # toBool: ETReal rounds half away from zero, ETInt tests != 0
    extra = [0.5, -0.5, 1.5, -1.5, 2.5, 0.49999999999999994, -0.49999999999999994, 0.5000000000000001, 1e-300, -1e-300]
    fvals = [p[0] for p in pairs] + extra * 7
    ivals = [EO.INT64_POOL[i % len(EO.INT64_POOL)] for i in range(n)]
    for tp, vals, fn, lf, of in ((FLOAT64, fvals, V.to_bool_real, lib.tq_vec_filter_real, O.vec_filter_real),
                                 (INT64, ivals, V.to_bool_int, lib.tq_vec_filter_int, O.vec_filter_int)):
        k = len(vals)
        col = EO.column(vals, tp, EO.null_mask(rng, k))
        want = np.array([fn(v) for v in vals], dtype=np.uint8) & col.not_null()
        m = Mem(mem)
        try:
            tc = m.inp(col)
            ptr, get = m.sel(k)
            assert lf(k, C.byref(tc), ptr, mem) == 0
            assert np.array_equal(get(), want)
        finally:
            m.free()
        assert np.array_equal(of(col), want)


@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("ua", [False, True])
def test_vec_in_int_mixed_signedness(lib, ua, mem):
    """x IN (l0 BIGINT, l1 BIGINT UNSIGNED): equal 64-bit patterns of different signedness are not equal values"""
    rng = np.random.default_rng(5 + ua)
    n = 64 * 40 + 63
    pick = lambda choices: choices[int(rng.integers(0, len(choices)))]   # noqa: E731
    x = [pick(EO.pool(ua)) for _ in range(n)]
    # each list item: x's 64-bit pattern read as the item's type, x's value where the type holds it, or a pool value
    l0 = [pick([V.i64(v), v if v <= V.I64_MAX else V.i64(v), pick(EO.INT64_POOL)]) for v in x]
    l1 = [pick([V.u64(v), v if v >= 0 else V.u64(v), pick(EO.UINT64_POOL)]) for v in x]
    a, c0, c1 = (EO.column(x, _tp(ua), EO.null_mask(rng, n, 0.1)), EO.column(l0, INT64, EO.null_mask(rng, n, 0.1)),
                 EO.column(l1, UINT64, EO.null_mask(rng, n, 0.1)))
    want, want_nn = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=bool)
    an, n0, n1 = a.not_null(), c0.not_null(), c1.not_null()
    for i in range(n):
        if not an[i]:
            continue
        r = V.in_int(x[i], ua, [(l0[i] if n0[i] else None, False), (l1[i] if n1[i] else None, True)])
        want_nn[i] = r is not None
        want[i] = r or 0
    m = Mem(mem)
    try:
        ta = m.inp(a)
        lst = (L.TQColumn * 2)(m.inp(c0), m.inp(c1))
        to, get = m.out(INT64, n)
        assert lib.tq_vec_in_int(n, C.byref(ta), int(ua), 2, lst, (C.c_int32 * 2)(0, 1), C.byref(to), mem) == 0
        assert_values(get(), want, want_nn)
    finally:
        m.free()
    assert_values(O.vec_in_int(a, [c0, c1])[1], want, want_nn)


# ------------------------------------------------------------------ tq_expr_eval
def expr_eval(prog, cols, mem):
    """-> (status, outputs, selected, warnings) of ExprProgram prog over host or device columns"""
    n = cols[0].length
    if mem == HOST:
        try:
            outs, sel, warn = prog.run(cols)
            return 0, outs, sel, warn
        except L.TQError as e:
            return e.status, None, None, None
    m = Mem(mem)
    try:
        ins = (L.TQColumn * len(cols))(*[m.inp(c) for c in cols])
        outs = [m.out(tp, n) for tp in prog.out_types]
        ops = (L.TQExprOp * max(len(prog.ops), 1))(*prog.ops)
        regs = (C.c_int32 * max(len(outs), 1))(*prog.out_regs)
        sel_ptr, get_sel = m.sel(n)
        dz = C.c_int64(0)
        st = L.load().tq_expr_eval(n, len(cols), ins, len(prog.ops), ops, len(outs), regs, (L.TQColumn * max(len(outs), 1))(*[o[0] for o in outs]),
                                   C.c_void_p(sel_ptr), C.byref(dz), mem)
        if st:
            return st, None, None, None
        return 0, [o[1]() for o in outs], get_sel(), dz.value
    finally:
        m.free()


def _one_op(spec):
    a, b = Col(0, _et(spec.ta)), Col(1, _et(spec.tb))
    return spec.expr(a, b)


@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("spec", SPECS, ids=repr)
def test_expr_eval_one_op(lib, spec, mem):
    op = _one_op(spec)
    flag_of = lambda n: Column(INT64, np.ones(n, dtype=np.int64))   # noqa: E731
    for n_mod in (1, 63):                                              # values, as a projection behind a passing filter
        a, b, want, want_nn, warn = value_rows(spec, n_mod)
        st, outs, sel, w = expr_eval(ExprProgram(3, [Col(2)], [op]), [a, b, flag_of(a.length)], mem)
        assert st == 0 and sel.all() and w == warn
        assert_values(outs[0], want, want_nn)
    smp = samples(spec)
    for x, y, kind, tag in smp:
        for pos, n in positions(129, mem):
            a, b = error_rows(spec, x, y, pos, n)
            assert expr_eval(ExprProgram(2, [], [op]), [a, b], mem)[0] == kind, (tag, pos)
            if pos in (0, n - 1):                                      # as a filter item, and behind a passing filter
                assert expr_eval(ExprProgram(2, [Func("isnull", op)], []), [a, b], mem)[0] == kind, (tag, pos)
    # the sampled rows together: an operand NULL, or removed by an earlier filter item / the Selection, raise nothing
    n = 64 * len(smp) + 63
    a, b = error_rows(spec, smp[0][0], smp[0][1], 0, n)
    flag = np.ones(n, dtype=np.int64)
    for k, (x, y, _, _) in enumerate(smp):
        a.values[64 * k], b.values[64 * k] = x, y
        flag[64 * k] = 0
    na = flag != 0
    assert expr_eval(ExprProgram(2, [], [op]), [Column(spec.ta, a.values, na), b], mem)[0] == 0
    if spec.kind != "neg":
        assert expr_eval(ExprProgram(2, [], [op]), [a, Column(spec.tb, b.values, na)], mem)[0] == 0
    fl = Column(INT64, flag)
    assert expr_eval(ExprProgram(3, [Col(2), Func("isnull", op)], []), [a, b, fl], mem)[0] == 0   # an earlier CNF item
    st, outs, sel, _ = expr_eval(ExprProgram(3, [Col(2)], [op]), [a, b, fl], mem)                 # Selection -> Projection
    assert st == 0 and np.array_equal(sel, na.astype(np.uint8))
    fr = Column(FLOAT64, np.where(na, 1.0, 0.49999999999999994))                                    # ETReal toBool removes it
    assert expr_eval(ExprProgram(3, [Col(2, "real")], [op]), [a, b, fr], mem)[0] == 0


@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
def test_expr_eval_compare_in_filter_edges(lib, mem):
    """comparisons of every sign mix, IN over mixed signedness and both toBool kinds as one-op programs"""
    rng = np.random.default_rng(8)
    for ua, ub in EO.INT_MIXES:
        pairs = _cmp_pairs(ua, ub)
        n = ((len(pairs) + 63) // 64) * 64 + 1
        pairs = (pairs * 2)[:n]
        a = EO.column([p[0] for p in pairs], _tp(ua), EO.null_mask(rng, n))
        b = EO.column([p[1] for p in pairs], _tp(ub), EO.null_mask(rng, n))
        nn = a.not_null() & b.not_null()
        A, B = Col(0, _et(_tp(ua))), Col(1, _et(_tp(ub)))
        projs = [Func(nm, A, B) for nm in ("lt", "le", "gt", "ge")]
        st, outs, _, _ = expr_eval(ExprProgram(2, [], projs), [a, b], mem)
        assert st == 0
        for op, got in enumerate(outs):
            assert_values(got, np.array([V.cmp_result(op, V.compare_int(x, y, ua, ub)[0]) for x, y in pairs], dtype=np.uint64), nn)
        st, outs, _, _ = expr_eval(ExprProgram(2, [], [Func("eq", A, B), Func("ne", A, B), Func("in", A, B, Const(None))]), [a, b], mem)
        assert st == 0
        for op, got in zip((4, 5), outs):
            assert_values(got, np.array([V.cmp_result(op, V.compare_int(x, y, ua, ub)[0]) for x, y in pairs], dtype=np.uint64), nn)
        an = a.not_null()
        win = [V.in_int(x, ua, [(y if bn else None, ub), (None, False)]) if xn else None for (x, y), xn, bn in zip(pairs, an, b.not_null())]
        assert_values(outs[2], np.array([w or 0 for w in win], dtype=np.uint64), np.array([w is not None for w in win]))
        # ETInt FILTER on the comparison: NULL stays in the set but is not selected
        st, _, sel, _ = expr_eval(ExprProgram(2, [Func("ge", A, B)], []), [a, b], mem)
        assert st == 0
        assert np.array_equal(sel, (np.array([V.cmp_result(3, V.compare_int(x, y, ua, ub)[0]) for x, y in pairs]) & nn).astype(np.uint8))
    vals = EO.FLOAT64_FILTER_POOL + [1.5, -1.5, 2.5, -2.5]
    col = EO.column((vals * 40)[: 64 * 2 + 63], FLOAT64, EO.null_mask(rng, 64 * 2 + 63))
    st, _, sel, _ = expr_eval(ExprProgram(1, [Col(0, "real")], []), [col], mem)
    assert st == 0
    assert np.array_equal(sel, np.array([V.to_bool_real(v) for v in col.values], dtype=np.uint8) & col.not_null())
    icol = EO.column((EO.INT64_POOL * 10)[: 64 * 3 + 1], INT64, EO.null_mask(rng, 64 * 3 + 1))
    st, _, sel, _ = expr_eval(ExprProgram(1, [Col(0)], []), [icol], mem)
    assert st == 0 and np.array_equal(sel, (icol.values != 0).astype(np.uint8) & icol.not_null())


def _edge_inputs(rng, n):
    """8 input columns of pool values (NULLs included): s0 s1 BIGINT, u0 u1 BIGINT UNSIGNED, d0 d1 d2 DOUBLE, f flag"""
    cols = [EO.column([EO.INT64_POOL[i] for i in rng.integers(0, len(EO.INT64_POOL), n)], INT64, EO.null_mask(rng, n, 0.1)) for _ in range(2)]
    cols += [EO.column([EO.UINT64_POOL[i] for i in rng.integers(0, len(EO.UINT64_POOL), n)], UINT64, EO.null_mask(rng, n, 0.1)) for _ in range(2)]
    cols += [EO.column([EO.FLOAT64_POOL[i] for i in rng.integers(0, len(EO.FLOAT64_POOL), n)], FLOAT64, EO.null_mask(rng, n, 0.1)) for _ in range(3)]
    cols.append(Column(INT64, rng.integers(0, 3, n)))
    return cols


def _limit_program():
    """8 inputs, 32 ops, 4 outputs"""
    S0, S1, U0, U1 = Col(0), Col(1), Col(2, "uint"), Col(3, "uint")
    D0, D1, D2, F = Col(4, "real"), Col(5, "real"), Col(6, "real"), Col(7)
    filters = [Func("or", Func("lt", Func("plus", S0, S1), Const(0)), Func("ge", Func("mul", U0, U1), Const(5, "uint"))),
               Func("not", Func("eq", Func("minus", D0, D1), Const(0.0, "real"))), F]
    projections = [Func("if", Func("gt", S0, S1), Func("neg", S0), Func("minus", S1, S0)), Func("ifnull", Func("plus", U0, S1), Func("mul", U1, Const(2, "uint"))),
                   Func("div", Func("plus", D0, D2), Func("mul", D1, D2)), Func("in", S0, U0, Const(-1))]
    prog = ExprProgram(8, filters, projections)
    while len(prog.ops) < 32:   # pad with repeated flag items (one FILTER op each) up to the limit
        filters.insert(0, F)
        prog = ExprProgram(8, filters, projections)
    assert len(prog.ops) == 32 and len(prog.out_regs) == 4
    return filters, projections


def _in_set_safe_rows(cols, filters, projections):
    """rows on which the oracle composition raises nothing when evaluated alone"""
    keep = []
    for i in range(cols[0].length):
        one = [Column(c.tp, c.values[i:i + 1], c.not_null()[i:i + 1]) for c in cols]
        try:
            oracle_select_project(one, filters, projections)
            keep.append(i)
        except OracleError:
            pass
    return np.array(keep)


def test_expr_eval_composed_and_limit_programs(lib):
    """composed programs over edge columns: the rows that raise nothing bit-exact against the oracle's builtins composed the
    way VecEvalBool composes them, and the whole column's error kind"""
    rng = np.random.default_rng(11)
    cols = _edge_inputs(rng, 700)
    S0, S1, U0, D0, D1 = Col(0), Col(1), Col(2, "uint"), Col(4, "real"), Col(5, "real")
    programs = [([Func("gt", Func("minus", S0, S1), Const(0))], [Func("mul", S0, Const(2)), Func("plus", U0, S1)]),
                ([Func("plus", D0, D1)], [Func("neg", Func("minus", S1, S0)), Func("div", D0, D1)]),
                ([], [Func("if", Func("lt", S0, Const(0)), Func("neg", S0), Func("mul", S0, S1))]),
                _limit_program()]
    for filters, projections in programs:
        check(cols, filters, projections)                 # the error kind of the whole column (or the values)
        keep = _in_set_safe_rows(cols, filters, projections)
        sub = [Column(c.tp, c.values[keep], c.not_null()[keep]) for c in cols]
        assert sub[0].length > 100
        assert check(sub, filters, projections) is not None


# ------------------------------------------------------------------ error order
I64_BIG, U64_BIG, D_BIG = -(1 << 62) - 1, 1 << 63, 1e300


def _order_cols(n=129, pos=64):
    """s: BIGINT whose sum with itself overflows at row pos, u: BIGINT UNSIGNED likewise, d: DOUBLE whose square overflows"""
    s = np.ones(n, dtype=np.int64)
    u = np.ones(n, dtype=np.uint64)
    d = np.ones(n)
    s[pos], u[pos], d[pos] = I64_BIG, U64_BIG, D_BIG
    return [Column(INT64, s), Column(UINT64, u), Column(FLOAT64, d)]


def order_cases(S, U, D):
    """(filters, projections, status) over Expr columns S (BIGINT), U (BIGINT UNSIGNED), D (DOUBLE): two or more ops raise
    different kinds on the same in-set row, the first in evaluation order decides"""
    ss, uu, dd = Func("plus", S, S), Func("plus", U, U), Func("mul", D, D)
    gt = lambda e: Func("gt", e, Const(0, e.tp))   # noqa: E731
    big, ubig, dbig = L.TQ_ERR_OVERFLOW_BIGINT, L.TQ_ERR_OVERFLOW_BIGINT_UNSIGNED, L.TQ_ERR_OVERFLOW_DOUBLE
    return [
        ([Func("and", gt(ss), gt(uu))], [], big),                                   # within one filter item
        ([Func("and", gt(uu), gt(ss))], [], ubig),
        ([Func("or", gt(dd), gt(uu))], [], dbig),
        ([gt(ss), gt(uu)], [], big),                                               # across CNF items
        ([gt(uu), gt(dd)], [], ubig),
        ([gt(dd), gt(ss)], [], dbig),
        ([Func("if", Const(1), Const(1), gt(ss)), gt(uu)], [], big),               # an op of the branch IF does not take
        ([Func("and", Func("if", Const(0), gt(ss), Const(1)), gt(uu))], [], big),
        ([Func("and", Func("and", gt(ss), gt(uu)), Func("lt", ss, Const(0)))], [], big),   # a CSE'd subtree: its first use
        ([Func("and", gt(uu), Func("and", gt(ss), Func("ne", uu, Const(1, "uint"))))], [], ubig),
    ], [
        ([], [ss, uu], big),                                                       # across projections
        ([], [uu, ss], ubig),
        ([], [dd, uu, ss], dbig),
        ([], [Func("mul", S, S), uu], big),
        ([], [Func("if", Const(1), Const(0), ss), uu], big),
        ([], [gt(ss), uu, ss], big),                                              # CSE'd across projections
        ([gt(uu)], [ss], ubig),                                                   # filter before projection
        ([Func("ne", S, Const(5))], [dd, ss], dbig),
    ]


@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
def test_expr_eval_error_order(lib, mem):
    cols = _order_cols()
    filt, proj = order_cases(Col(0), Col(1, "uint"), Col(2, "real"))
    for filters, projections, status in filt + proj:
        assert expr_eval(ExprProgram(3, filters, projections), cols, mem)[0] == status, (filters, projections)
        if mem == HOST:
            assert check(cols, filters, projections) is None      # the oracle composition agrees


# ------------------------------------------------------------------ the joins' programs
def edge_tables(spec, x, y, ni=None, nulls=None, flag0=None, want=None):
    """inner row i joins outer row i by key: inner column a = x[i], outer column b = y[i], w = 1 (0 on rows flag0), want = the
    expected result column.  ni > len(x): extra inner rows whose keys match nothing (the hash join's partitioned path from 2^18
    build rows).  nulls = (a NULL, b NULL) masks over the joined rows."""
    n = len(x)
    ni = ni or n
    ik = np.concatenate([np.arange(n), np.arange(n, ni) + (1 << 40)]).astype(np.int64)
    nn_a, nn_b = np.ones(ni, dtype=bool), np.ones(n, dtype=bool)
    if nulls is not None:
        nn_a[:n] &= ~nulls[0]
        nn_b &= ~nulls[1]
    flag = np.ones(n, dtype=np.int64)
    if flag0 is not None:
        flag[flag0] = 0
    inner = {"ik": Column(INT64, ik), "a": Column(spec.ta, np.resize(EO.np_values(x, spec.ta), ni), nn_a)}
    outer = {"ok": Column(INT64, np.arange(n, dtype=np.int64)), "b": Column(spec.tb, EO.np_values(y, spec.tb), nn_b), "w": Column(INT64, flag)}
    if want is not None:
        outer["want"] = want
    return TJ.Tables(True, inner, outer)


def join_status(kind, t, prog, jt=INNER_JOIN, sel=None):
    try:
        TJ.run(kind, jt, t.oir, t.it, t.ic, t.ot, t.oc, [0], [0], prog, sel=sel)
        return 0
    except L.TQError as e:
        return e.status


def _prog(spec, t):
    return [Func("isnull", spec.expr(t.col("a"), t.col("b")))]


def join_values(kind, spec, ni=None):
    """the edge rows the restatement lets through as key-matched pairs; the program keeps the rows whose result equals the
    restatement's value, so every non-NULL result survives; the rows and the warnings equal the oracle's"""
    xs, ys, res = rows_of(spec)
    ok = [i for i, r in enumerate(res) if r[1] is None]
    n = ((len(ok) + 63) // 64) * 64 + 1
    idx = (ok * 2)[:n]
    want = [res[i][0] for i in idx]
    if spec.kind == "real":
        wc = Column(FLOAT64, np.array([0.0 if v is None else v for v in want]), np.array([v is not None for v in want]))
    else:
        wc = Column(spec.out_tp, np.array(want, dtype=np.uint64).view(np.int64 if spec.out_tp == INT64 else np.uint64))
    t = edge_tables(spec, [xs[i] for i in idx], [ys[i] for i in idx], ni, want=wc)
    prog = [Func("eq", spec.expr(t.col("a"), t.col("b")), t.col("want"))]
    got, _ = TJ.check(kind, t, prog, INNER_JOIN, ordered=kind == "merge")
    assert got.num_rows() == sum(v is not None for v in want)
    if spec.kind == "real":    # the result itself as an ETReal item: toBool rounds half away from zero
        TJ.check(kind, t, [spec.expr(t.col("a"), t.col("b"))], INNER_JOIN, ordered=kind == "merge")


def join_errors(kind, spec, ni=None, pos_list=(0, 63, 64, 128)):
    xs, ys, res = rows_of(spec)
    ok = [i for i, r in enumerate(res) if r[1] is None]
    n = 129
    base_x, base_y = [xs[i] for i in (ok * 2)[:n]], [ys[i] for i in (ok * 2)[:n]]
    smp = samples(spec)
    for x, y, kind_, tag in smp:
        for pos in pos_list:
            bx, by = list(base_x), list(base_y)
            bx[pos], by[pos] = x, y
            t = edge_tables(spec, bx, by, ni)
            assert join_status(kind, t, _prog(spec, t)) == kind_, (tag, pos)
    # every sample at once: with an operand NULL, behind an earlier item that drops the row, outside the outer filter
    bx, by = list(base_x), list(base_y)
    rows = [1 + 2 * k for k in range(len(smp))]
    for r, (x, y, _, _) in zip(rows, smp):
        bx[r], by[r] = x, y
    on, off = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
    on[rows] = True
    for nulls in ((on, off), (off, on))[: 1 if spec.kind == "neg" else 2]:
        t = edge_tables(spec, bx, by, ni, nulls=nulls)
        assert join_status(kind, t, _prog(spec, t)) == 0
    t = edge_tables(spec, bx, by, ni, flag0=rows)
    assert join_status(kind, t, [Func("ne", t.col("w"), Const(0))] + _prog(spec, t)) == 0
    assert join_status(kind, t, _prog(spec, t), sel=(~on).astype(np.uint8)) == 0


JOIN_SITES = [("hash", None), ("hash", 270000), ("merge", None)]


@pytest.mark.parametrize("site", JOIN_SITES, ids=["hash-one-table", "hash-partitioned", "merge"])
@pytest.mark.parametrize("spec", SPECS, ids=repr)
def test_join_program_edges(lib, spec, site):
    kind, ni = site
    join_values(kind, spec, ni)
    join_errors(kind, spec, ni, (0, 128) if ni else (0, 63, 64, 128))


def _order_tables(jt):
    """one key-matched row: inner is = iu = the overflowing operands, outer os / ou / od likewise; plus a row that only joins"""
    inner = {"ik": Column(INT64, [1, 2]), "is": Column(INT64, [I64_BIG, 1]), "iu": Column(UINT64, np.array([U64_BIG, 1], dtype=np.uint64)),
             "id": Column(FLOAT64, [D_BIG, 1.0])}
    outer = {"ok": Column(INT64, [1, 2]), "os": Column(INT64, [I64_BIG, 1]), "ou": Column(UINT64, np.array([U64_BIG, 1], dtype=np.uint64)),
             "od": Column(FLOAT64, [D_BIG, 1.0])}
    return TJ.Tables(False, inner, outer)


def join_error_order(kind, jt=INNER_JOIN):
    t = _order_tables(jt)
    S, U, D = t.col("is"), t.col("iu"), t.col("id")
    filt, _ = order_cases(S, U, D)
    so, uo = t.col("os"), t.col("ou")
    gt = lambda e: Func("gt", e, Const(0, e.tp))   # noqa: E731
    cases = filt + [([Func("and", gt(Func("plus", S, so)), gt(Func("plus", U, uo)))], [], L.TQ_ERR_OVERFLOW_BIGINT),
                    ([Func("and", gt(Func("plus", U, uo)), gt(Func("plus", S, so)))], [], L.TQ_ERR_OVERFLOW_BIGINT_UNSIGNED)]
    for filters, _, status in cases:
        assert join_status(kind, t, filters, jt) == status, filters
        assert TJ.check(kind, t, filters, jt)[0] is None          # the oracle composition raises the same kind


@pytest.mark.parametrize("kind", ["hash", "merge"])
@pytest.mark.parametrize("jt", [INNER_JOIN, LEFT_OUTER_JOIN])
def test_join_program_error_order(lib, kind, jt):
    join_error_order(kind, jt)
