"""The key-less hash join on the CPU: the oracle (every build row in one chain) against the numpy nested loop, and the
reference's key-less cases (executor/join_test.go)."""
import numpy as np
import pytest

from keyless_oracle import keyless_hash_join, keyless_join_with_program, nested_loop
from tinysql_b200.chunk import BYTES, FLOAT32, FLOAT64, INT64, Column
from tinysql_b200.executor import INNER_JOIN, LEFT_OUTER_JOIN, RIGHT_OUTER_JOIN
from tinysql_b200.expression import Col, Const, Func
from util import assert_same_ordered

LT = 0
# (join type, outer_is_right)
SHAPES = [(INNER_JOIN, False), (INNER_JOIN, True), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)]


def _sides(rng, nb, npr):
    """build: v INT64 (NULLs), s BYTES, f FLOAT32; probe: v INT64 (NULLs), d FLOAT64"""
    bt = [INT64, BYTES, FLOAT32]
    bc = [Column(INT64, rng.integers(0, 50, nb), rng.random(nb) > 0.1),
          Column(BYTES, [None if rng.random() < 0.1 else b"s%d" % rng.integers(0, 1000) for _ in range(nb)]),
          Column(FLOAT32, rng.random(nb).astype(np.float32), rng.random(nb) > 0.2)]
    pt = [INT64, FLOAT64]
    pc = [Column(INT64, rng.integers(0, 50, npr), rng.random(npr) > 0.1), Column(FLOAT64, rng.random(npr))]
    return bt, bc, pt, pc


def _lt_build_probe(bc, pc):
    """B.v < P.v with NULL failing"""
    bv, bn, pv, pn = bc[0].values, bc[0].not_null(), pc[0].values, pc[0].not_null()
    return lambda pi, bi: bn[bi] & pn[pi] & (bv[bi] < pv[pi])


@pytest.mark.parametrize("nb", [0, 1, 31, 32, 33, 1000])
@pytest.mark.parametrize("jt,oir", SHAPES)
@pytest.mark.parametrize("with_cond", [False, True])
def test_oracle_keyless_matches_nested_loop(nb, jt, oir, with_cond):
    rng = np.random.default_rng(nb * 7 + jt * 3 + oir + 11 * with_cond)
    npr = 40
    bt, bc, pt, pc = _sides(rng, nb, npr)
    sel = rng.random(npr) > 0.25
    dflt = [7, None, None] if jt != INNER_JOIN else None
    n_left = len(bt) if oir else len(pt)
    bv_out, pv_out = (0, n_left) if oir else (n_left, 0)
    conds = [(LT, bv_out, pv_out)] if with_cond else []
    got = keyless_hash_join(jt, oir, bt, bc, pt, pc, sel, conds, dflt)
    want = nested_loop(jt, oir, bc, pc, sel, _lt_build_probe(bc, pc) if with_cond else None, dflt)
    assert_same_ordered(got, want)


PROGRAMS = [
    # comparisons: B.v < P.v AND B.f > 0.25 (as DOUBLE input: probe d)
    lambda bvo, pvo, pdo: [Func("lt", Col(bvo), Col(pvo)), Func("gt", Col(pdo, "real"), Const(0.25, "real"))],
    # arithmetic: B.v + P.v >= 60
    lambda bvo, pvo, pdo: [Func("ge", Func("plus", Col(bvo), Col(pvo)), Const(60))],
    # IF / IN: IF(P.v > 25, B.v IN (1, 2, 3), B.v = P.v)
    lambda bvo, pvo, pdo: [Func("if", Func("gt", Col(pvo), Const(25)), Func("in", Col(bvo), Const(1), Const(2), Const(3)), Func("eq", Col(bvo), Col(pvo)))],
]


def _program_passes(k, bc, pc):
    bv, bn, pv, pn, pd = bc[0].values, bc[0].not_null(), pc[0].values, pc[0].not_null(), pc[1].values
    if k == 0:
        return lambda pi, bi: bn[bi] & pn[pi] & (bv[bi] < pv[pi]) & (pd[pi] > 0.25)
    if k == 1:
        return lambda pi, bi: bn[bi] & pn[pi] & (bv[bi] + pv[pi] >= 60)

    def f(pi, bi):
        take_in = pn[pi] & (pv[pi] > 25)
        in_ok = bn[bi] & np.isin(bv[bi], [1, 2, 3])
        eq_ok = bn[bi] & pn[pi] & (bv[bi] == pv[pi])
        return np.where(take_in, in_ok, eq_ok)
    return f


@pytest.mark.parametrize("k", range(len(PROGRAMS)))
@pytest.mark.parametrize("jt,oir", SHAPES)
def test_join_program_keyless_matches_nested_loop(k, jt, oir):
    rng = np.random.default_rng(100 + k * 5 + jt * 2 + oir)
    bt, bc, pt, pc = _sides(rng, 45, 60)
    bt, bc = bt[:1], bc[:1]   # condition inputs are BIGINT / DOUBLE columns
    sel = rng.random(60) > 0.2
    n_left = len(bt) if oir else len(pt)
    bvo, pvo, pdo = (0, n_left, n_left + 1) if oir else (n_left, 0, 1)
    got, warn = keyless_join_with_program(jt, oir, bt, bc, pt, pc, PROGRAMS[k](bvo, pvo, pdo), sel)
    want = nested_loop(jt, oir, bc, pc, sel, _program_passes(k, bc, pc))
    assert warn == 0
    assert_same_ordered(got, want)


def test_reference_hash_join_encode_decode_row():
    """join_test.go:318-329 TestHashJoinExecEncodeDecodeRow: `select ts from t1 inner join t2 where t2.name = 'xxx'` — the WHERE
    on t2 alone is pushed below the join, which keeps no equality: a key-less inner join with a var-len build payload."""
    t1 = [Column(INT64, [1])]
    t2 = [Column(INT64, [1]), Column(BYTES, [b"xxx"]), Column(BYTES, [b"2003-06-09 10:51:26"])]
    got = keyless_hash_join(INNER_JOIN, False, [INT64, BYTES, BYTES], t2, [INT64], t1)
    assert [r[3] for r in got.rows()] == [b"2003-06-09 10:51:26"]


def test_reference_embedded_outer_join():
    """join_test.go:392-401 TestEmbeddedOuterJoin: the outer left join's `ON t2.b = 1` names only the outer side
    ((t1 left join t2) = {(1, 1, NULL, NULL)}), so it arrives as selected[] = [0]; the inner side (t3 left join t4) is empty."""
    outer = [Column(INT64, [1]), Column(INT64, [1]), Column(INT64, [0], [False]), Column(INT64, [0], [False])]
    inner = [Column(INT64, np.zeros(0, dtype=np.int64)) for _ in range(4)]
    got = keyless_hash_join(LEFT_OUTER_JOIN, False, [INT64] * 4, inner, [INT64] * 4, outer, selected=[0])
    assert got.rows() == [(1, 1, None, None, None, None, None, None)]


def test_reference_inject_proj_on_top_n():
    """join_test.go:403-414 TestInjectProjOnTopN: `select t1.a+t1.b as result from t1 left join t2 on 1 = 0`: an outer join on
    an empty build side."""
    t1 = [Column(INT64, [1]), Column(INT64, [1])]
    t2 = [Column(INT64, np.zeros(0, dtype=np.int64)) for _ in range(2)]
    got = keyless_hash_join(LEFT_OUTER_JOIN, False, [INT64, INT64], t2, [INT64, INT64], t1)
    assert [r[0] + r[1] for r in got.rows()] == [2]
    assert got.rows() == [(1, 1, None, None)]
