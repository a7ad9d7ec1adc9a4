"""CPU suite: the fixed-width builtins at their overflow and sign boundaries.

The restatement of the reference's per-row statements (vec_statements.py) against the oracle (oracle/oracle.c) row by row over
the edge operands of edge_operands.py, for every op and sign mix; against the exact-range row model of test_expr_oracle_twin.py
wherever none of the reference's quirks decides the row.  Then the merge-join program cases of test_gpu_builtin_edges.py run
against the emulation build of tests/emu (sort.cu's k_mj_prog and the interpreter of expr_prog.cuh), as
test_emu_join_program.py does."""
import numpy as np
import pytest

import edge_operands as EO
import oracle_py as O
import test_gpu_builtin_edges as TB
import vec_statements as V
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)
from test_expr_oracle_twin import row_arith_int
from tinysql_b200.chunk import FLOAT64, INT64, UINT64, Column
from tinysql_b200.executor import INNER_JOIN, LEFT_OUTER_JOIN


def _one(vals, tp):
    return EO.column(vals, tp)


def quirk(op, x, y, ua, ub):
    """the rows where the reference's check is not the exact range test: plusUS compares lh with itself, minusSU tests
    lh - MinInt64 < rh, minusSS wraps -MinInt64, MultiplyInt's wrapped quotient hides -1 * MinInt64"""
    lh, rh = V.i64(x), V.i64(y)
    if op == 0 and ua and not ub:
        return rh > 0 and (V.u64(lh) > V.U64_MAX - V.u64(lh)) != (V.u64(lh) > V.U64_MAX - rh)
    if op == 1 and ub and not ua:
        return (V.u64(V.i64(lh - V.I64_MIN)) < V.u64(rh)) != (x < y)
    if op == 1 and not ua and not ub:
        return rh == V.I64_MIN
    if op == 2 and not ua and not ub:
        return (lh, rh) == (-1, V.I64_MIN)
    return False


def _check_against_oracle(spec):
    xs, ys, res = TB.rows_of(spec)
    # the rows that raise nothing, in one call, with NULL rows holding raising operands
    for n_mod in (1, 63):
        a, b, want, want_nn, warn = TB.value_rows(spec, n_mod)
        rc, out, dz = TB.oracle_call(spec, a, b)
        assert rc == 0 and dz == warn
        TB.assert_values(out, want, want_nn)
    # every raising row alone
    for x, y, (_, kind, tag) in zip(xs, ys, res):
        if kind is None:
            continue
        a, b = _one([x], spec.ta), _one([y], spec.tb)
        assert TB.oracle_call(spec, a, b)[0] == kind, (spec, x, y, tag)
    return {t for _, k, t in res if k is not None}


@pytest.mark.parametrize("spec", TB.SPECS, ids=repr)
def test_restatement_equals_oracle(spec):
    tags = _check_against_oracle(spec)
    assert tags == spec.raising_tags()


@pytest.mark.parametrize("op", [0, 1, 2])
@pytest.mark.parametrize("ua,ub", EO.INT_MIXES)
def test_restatement_equals_exact_range_outside_the_quirks(op, ua, ub):
    xs, ys, res = TB.rows_of(TB.Spec("int", op, ua, ub))
    tps = (UINT64 if ua else INT64, UINT64 if ub else INT64)
    quirks = 0
    for x, y, (v, kind, tag) in zip(xs, ys, res):
        if quirk(op, x, y, ua, ub):
            quirks += 1
            continue
        want, err = row_arith_int(op, _one([x], tps[0]), _one([y], tps[1]), 0)
        assert err == (kind is not None), (x, y, tag)
        if not err:
            assert V.u64(want) == v
    # the quirky mixes do meet their quirks at these edges
    assert (quirks > 0) == ((op, ua, ub) in {(0, True, False), (1, False, True), (1, False, False), (2, False, False)})


def test_quirks_of_the_reference():
    assert V.plus_int(1 << 63, 1, True, False)[1] == V.UBIGINT                # plusUS: 2^63 + 1 fits, lh + lh does not
    assert V.plus_int((1 << 63) - 1, 1 << 62, True, False)[1] is None
    assert V.minus_int(0, V.I64_MIN, False, False)[1] is None                  # minusSS: 0 - MinInt64 overflows unreported
    assert V.minus_int(-1, V.I64_MIN, False, False)[1] == V.BIGINT             # ... and -1 - MinInt64 fits but raises
    assert V.minus_int(0, 1, False, True)[1] is None                           # minusSU: 0 - 1 as BIGINT UNSIGNED unreported
    assert V.mul_int(-1, V.I64_MIN, False, False) == (V.u64(V.I64_MIN), None, None)
    assert V.mul_int(V.I64_MIN, -1, False, False)[1] == V.BIGINT
    assert V.plus_real(V.DBL_MAX, 1.0)[1] == V.DOUBLE                         # the sum rounds to DBL_MAX, the check raises
    assert V.plus_real(V.DBL_MAX / 2, V.DBL_MAX / 2) == (V.DBL_MAX, None, None)
    assert V.to_bool_real(0.49999999999999994) == 0 and V.to_bool_real(-0.5) == 1 and V.to_bool_real(float("nan")) == 1


@pytest.mark.parametrize("ua,ub", EO.INT_MIXES)
def test_compare_int_restatement_equals_oracle_and_exact(ua, ub):
    pairs = TB._cmp_pairs(ua, ub)
    a = EO.column([p[0] for p in pairs], UINT64 if ua else INT64)
    b = EO.column([p[1] for p in pairs], UINT64 if ub else INT64)
    for op in range(6):
        want = np.array([V.cmp_result(op, V.compare_int(x, y, ua, ub)[0]) for x, y in pairs], dtype=np.uint64)
        exact = np.array([V.cmp_result(op, (x > y) - (x < y)) for x, y in pairs], dtype=np.uint64)   # the values compare exactly
        assert np.array_equal(want, exact)
        rc, out = O.vec_compare_int(op, a, b)
        assert rc == 0 and np.array_equal(out.raw(), want)


def test_compare_real_to_bool_and_in_restatement_equal_oracle():
    pool = EO.FLOAT64_FILTER_POOL
    pairs = [(x, y) for x in pool for y in pool]
    a, b = EO.column([p[0] for p in pairs], FLOAT64), EO.column([p[1] for p in pairs], FLOAT64)
    for op in range(6):
        want = np.array([V.cmp_result(op, V.compare_float(x, y)) for x, y in pairs], dtype=np.uint64)
        assert np.array_equal(O.vec_compare_real(op, a, b)[1].raw(), want)
    vals = pool + [1.5, -1.5, 2.5, -2.5, 0.5000000000000001]
    col = EO.column(vals, FLOAT64)
    assert list(O.vec_filter_real(col)) == [V.to_bool_real(v) for v in vals]
    icol = EO.column(EO.INT64_POOL, INT64)
    assert list(O.vec_filter_int(icol)) == [V.to_bool_int(v) for v in EO.INT64_POOL]
    for ua in (False, True):
        xs = EO.pool(ua)
        for lu in (False, True):
            for y in EO.pool(lu):
                a = EO.column(xs, UINT64 if ua else INT64)
                lst = [EO.column([y] * len(xs), UINT64 if lu else INT64), Column(INT64, np.zeros(len(xs), dtype=np.int64), np.zeros(len(xs), dtype=bool))]
                rc, out = O.vec_in_int(a, lst)
                want = [V.in_int(x, ua, [(y, lu), (None, False)]) for x in xs]
                assert rc == 0 and out.tolist() == want, (ua, lu, y)


# ------------------------------------------------------------------ the merge join's program on the emulation build
@pytest.mark.parametrize("spec", TB.SPECS, ids=repr)
def test_emu_merge_join_program_edges(emu, spec):
    TB.join_values("merge", spec)
    TB.join_errors("merge", spec, pos_list=(0, 63, 64, 128))


@pytest.mark.parametrize("jt", [INNER_JOIN, LEFT_OUTER_JOIN])
def test_emu_merge_join_program_error_order(emu, jt):
    """(is + os > 0) AND (iu + ou > 0) with both sums overflowing: the signed sum comes first, BIGINT"""
    TB.join_error_order("merge", jt)
