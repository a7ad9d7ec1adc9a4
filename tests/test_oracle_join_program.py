"""CPU suite: the restatement of the joiner's OtherConditions for the program form (join_program_oracle.py) is pinned to the
oracle's comparison form and to the reference's own known answers.

1. The program form of every comparison list the comparison-form tests use gives exactly O.hash_join(..., conds) /
   O.merge_join(..., conds) — the restatement composes the same filter / miss-row logic the oracle has for comparisons.
2. The reference goldens whose join carries a two-sided OtherCondition (tests/golden/reference_cases.json):
   inner_other_condition (executor/join_test.go:137-139) and self_join_sum_gt_5 (join_test.go:115-116: predicate push-down
   turns `a.c1 + b.c1 > 5` into an OtherCondition of the inner join — arithmetic inside the joiner).  join_test.go:82-83 is
   not one of them: its one-sided `t.c1 != 1` reaches the join as the outer filter."""
import json
import os

import numpy as np
import pytest

import oracle_py as O
from join_program_oracle import conds_to_program, join_with_program
from tinysql_b200.chunk import FLOAT64, INT64, UINT64, Column
from tinysql_b200.expression import Col, Const, Func
from util import assert_same_multiset, assert_same_ordered, gen_col

INNER, LEFT, RIGHT = 0, 1, 2
GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_cases.json")))


def out_types(oir, it, ot):
    return (list(it) + list(ot)) if oir else (list(ot) + list(it))


@pytest.mark.parametrize("jt,oir", [(INNER, False), (INNER, True), (LEFT, False), (RIGHT, True)])
def test_program_form_of_hash_join_comparisons_equals_the_oracle(jt, oir):
    """the tables and comparison lists of test_join_other_conditions / test_join_default_inner_row, at CPU sizes"""
    rng = np.random.default_rng(40 + jt + int(oir))
    nb, npr = 300, 2000
    ndv = nb // 3
    bcols = [gen_col(rng, INT64, nb, 0.05, 0, ndv), gen_col(rng, INT64, nb, 0.1, -50, 50), gen_col(rng, FLOAT64, nb, 0.1)]
    pcols = [gen_col(rng, FLOAT64, npr, 0.1), gen_col(rng, INT64, npr, 0.05, 0, ndv + 2), gen_col(rng, INT64, npr, 0.1, -50, 50)]
    bt, pt = [INT64, INT64, FLOAT64], [FLOAT64, INT64, INT64]
    conds = [(0, 1, 5), (3, 2, 3), (5, 5, None, INT64, 7)] if oir else [(0, 4, 2), (3, 5, 0), (5, 2, None, INT64, 7)]
    sel = (rng.random(npr) > 0.2).astype(np.uint8)
    for s in (None, sel):
        want = O.hash_join(jt, oir, bt, bcols, pt, pcols, [0], [1], s, conds)
        got, warn = join_with_program("hash", jt, oir, bt, bcols, pt, pcols, [0], [1], conds_to_program(conds, out_types(oir, bt, pt)), s)
        assert_same_multiset(got, want)
        assert warn == 0
    if jt != INNER:   # test_join_default_inner_row: b1 < p1 with defaultInner
        pcols2 = [gen_col(rng, INT64, npr, 0.05, 0, nb), gen_col(rng, INT64, npr, 0.1, -50, 50)]
        pt2 = [INT64, INT64]
        conds = [(0, 1, 3)] if oir else [(0, 3, 1)]
        defaults = [None, 0, 2.5]
        want = O.hash_join(jt, oir, bt, bcols, pt2, pcols2, [0], [0], None, conds, default_inner=defaults)
        got, _ = join_with_program("hash", jt, oir, bt, bcols, pt2, pcols2, [0], [0], conds_to_program(conds, out_types(oir, bt, pt2)),
                                   default_inner=defaults)
        assert_same_multiset(got, want)


@pytest.mark.parametrize("jt,oir", [(INNER, False), (LEFT, False), (RIGHT, True), (INNER, True)])
def test_program_form_of_merge_join_comparisons_equals_the_oracle(jt, oir):
    """the tables and comparison lists of test_merge_join_other_conditions, at CPU sizes; in order"""
    rng = np.random.default_rng(90 + jt + 3 * int(oir))
    ni, no = 2000, 3000
    it, ot = [INT64, INT64, FLOAT64], [INT64, UINT64, FLOAT64, INT64]
    ic = [Column(INT64, np.sort(rng.integers(0, ni // 4, ni))), gen_col(rng, INT64, ni, 0.1, -50, 50), Column(FLOAT64, rng.integers(0, 100, ni) * 0.5, rng.random(ni) > 0.1)]
    oc = [Column(INT64, np.sort(rng.integers(0, ni // 3, no))), gen_col(rng, UINT64, no, 0.1, 0, 50), Column(FLOAT64, rng.integers(0, 100, no) * 0.5), Column(INT64, np.arange(no))]
    sel = (rng.random(no) > 0.1).astype(np.uint8)
    n_left = len(it) if oir else len(ot)
    icol = lambda c: c if oir else n_left + c
    ocol = lambda c: n_left + c if oir else c
    for conds in ([(0, icol(1), ocol(1))], [(3, icol(2), ocol(2)), (5, icol(1), None, INT64, 7)], [(4, ocol(2), None, FLOAT64, 12.5)],
                  [(2, icol(1), None, INT64, 1000)]):
        want = O.merge_join(jt, oir, it, ic, ot, oc, [0], [0], sel, conds=conds)
        got, warn = join_with_program("merge", jt, oir, it, ic, ot, oc, [0], [0], conds_to_program(conds, out_types(oir, it, ot)), sel)
        assert_same_ordered(got, want)
        assert warn == 0


def _golden(name):
    return next(c for c in GOLDEN["join"] if c["name"] == name)


def _table(rows):
    return [Column(INT64, [r[i] for r in rows]) for i in range(len(rows[0]))]


@pytest.mark.parametrize("oir", [False, True])
def test_reference_golden_inner_other_condition(oir):
    """join_test.go:137-139: the inner join's OtherCondition `r[2] < r[1]` (t1.c1 < t.c2) over the output row t ++ t1"""
    case = _golden("inner_other_condition")
    lhs, rhs = _table(case["lhs"]), _table(case["rhs"])
    flt = [Func("lt", Col(2), Col(1))]
    # the build (inner) side is the right child unless outer_is_right; the output row is always lhs ++ rhs
    if oir:
        got, _ = join_with_program("hash", INNER, True, [INT64] * 2, lhs, [INT64] * 2, rhs, case["lkey"], case["rkey"], flt)
    else:
        got, _ = join_with_program("hash", INNER, False, [INT64] * 2, rhs, [INT64] * 2, lhs, case["rkey"], case["lkey"], flt)
    assert sorted(got.rows()) == sorted(tuple(r) for r in case["expect"])


@pytest.mark.parametrize("kind", ["hash", "merge"])
def test_reference_golden_self_join_sum_gt_5(kind):
    """join_test.go:115-116: `select a.c1 from t a, t b where a.c1 = b.c1 and a.c1 + b.c1 > 5` — the pushed-down WHERE term is an
    OtherCondition of the inner join, evaluated with BIGINT arithmetic inside the joiner"""
    case = _golden("self_join_sum_gt_5")
    lhs, rhs = _table(case["lhs"]), _table(case["rhs"])
    flt = [Func("gt", Func("plus", Col(0), Col(1)), Const(5))]
    got, warn = join_with_program(kind, INNER, False, [INT64], rhs, [INT64], lhs, case["rkey"], case["lkey"], flt)
    assert [tuple(r[i] for i in case["select"]) for r in got.rows()] == [tuple(r) for r in case["expect"]]
    assert warn == 0
