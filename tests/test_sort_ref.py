"""CPU suite: the exact sort / TopN / merge-join reference of tests/sort_ref.py and its aimed families.

Every family must have the property it is named after (its self-check), and the reference must agree with the oracle on
every family and with the reference's own known answers (SORT_CASES / MERGE_CASES): two restatements written in different
ways, so that a test of the kernels against either one means the same."""
import numpy as np
import pytest

import oracle_py as O
import sort_ref as R
from sort_cases import MERGE_CASES, SORT_CASES

SORTS = R.sort_families(np.random.default_rng(7))
MJS = R.mj_keys(np.random.default_rng(8)) + R.mj_unsorted()
JOINS = [(R.INNER, False), (R.LEFT, False), (R.RIGHT, True)]


@pytest.mark.parametrize("case", SORTS + MJS, ids=[c.name for c in SORTS + MJS])
def test_family_has_its_property(case):
    R.check_family([case])


@pytest.mark.parametrize("case", SORTS, ids=[c.name for c in SORTS])
def test_reference_sort_equals_oracle(case):
    cols = case.columns()
    for by, off, cnt in case.sorts:
        want = R.canon_rows(R.sort_rows(case.rows(), by, off, cnt))
        assert R.canon_rows(O.sort(case.types, cols, by, off, cnt).rows()) == want, (by, off, cnt)


@pytest.mark.parametrize("case", [c for c in MJS if not c.refused], ids=[c.name for c in MJS if not c.refused])
def test_reference_merge_join_equals_oracle(case):
    ic, oc = case.columns(), case.ocolumns()
    sel = [int(i % 3 != 1) for i in range(len(case.ocols[0]))]
    for jt, oir in JOINS:
        for s in (None, sel):
            want = R.canon_rows(R.mj_expect(case, jt, oir, s))
            got = O.merge_join(jt, oir, case.types, ic, case.otypes, oc, case.ik, case.ok, None if s is None else np.array(s, np.uint8))
            assert R.canon_rows(got.rows()) == want, (jt, oir, s is not None)


@pytest.mark.parametrize("case", SORT_CASES, ids=[c[0] for c in SORT_CASES])
def test_reference_sort_known_answers(case):
    _, types, cols, by, off, cnt, want = case
    rows = [tuple(r) for r in zip(*[c.tolist() for c in cols])]
    assert R.sort_rows(rows, by, off, cnt) == want


@pytest.mark.parametrize("case", MERGE_CASES, ids=[c[0] for c in MERGE_CASES])
def test_reference_merge_join_known_answers(case):
    _, jt, oir, it, ic, ot, oc, ik, ok, sel, want = case
    irows = [tuple(r) for r in zip(*[c.tolist() for c in ic])]
    orows = [tuple(r) for r in zip(*[c.tolist() for c in oc])]
    assert R.merge_join(jt, oir, irows, len(it), orows, ik, ok, sel) == want


def test_reference_default_inner_and_signedness():
    irows = [(1, 10), (3, 30)]
    orows = [(1,), (2,), (3,), (4,)]
    assert R.merge_join(R.LEFT, False, irows, 2, orows, [0], [0], default_inner=[None, 0]) == [(1, 1, 10), (2, None, 0), (3, 3, 30), (4, None, 0)]
    # BIGINT -1 and BIGINT UNSIGNED 2^64 - 1 share a bit pattern and are different values
    assert R.merge_join(R.INNER, False, [(-1,), (0,)], 1, [(0,), (R.UINT64_MAX,)], [0], [0]) == [(0, 0)]


def test_pass_count_restatement_by_hand():
    """the restated pass count on inputs small enough to count by hand"""
    from tinysql_b200.chunk import BYTES, FLOAT64, INT64
    assert R.passes([INT64], [[3, 3, 3]], [False], [(0, False)]) == 0
    assert R.passes([INT64], [[3, 4]], [False], [(0, False)]) == 1
    assert R.passes([INT64], [[-1, 0]], [False], [(0, True)]) == 8             # 0x7FFF.. against 0x8000..
    assert R.passes([INT64], [[3, 4]], [True], [(0, False)]) == 1              # a NULL flag word that is constant costs nothing
    assert R.passes([INT64], [[3, None]], [True], [(0, False)]) == 2 + 1       # 0x80..03 against 0 (bytes 0 and 7); the flag word
    assert R.passes([FLOAT64], [[0.0, -0.0]], [False], [(0, False)]) == 0      # the fold
    # "a" / "a\0": the chunk words agree, the length word differs in its low byte
    assert R.passes([BYTES], [[b"a", b"a\0"]], [False], [(0, False)]) == 1
    assert R.passes([BYTES], [[b"", b""]], [False], [(0, False)]) == 0
    assert R.passes([INT64], [[3, 4]], [False], [(0, False)], 2, 5) == 0        # an empty window sorts nothing
