"""Restatement of the joiner's OtherConditions for the program form (TEST INFRASTRUCTURE).

joiner.tryToMatchInners (executor/joiner.go:225-248,288-311) joins one outer row with its key-matched inner rows, filter
(joiner.go:155-167) keeps the joined rows expression.VectorizedFilter selects, and an outer row none of whose joined rows
survive goes to onMissMatch (joiner.go:274-277,337-340): an outer join emits it once with a NULL / defaultInner inner side.
An outer row without key matches, with a NULL key or outside the outer filter returns before filter (inners.Len() == 0), so
its conditions never run.

The key-matched pairs come from the oracle's own joins (O.hash_join / O.merge_join without conditions) with a row-id column
appended to each side; the conditions are evaluated with the oracle's per-builtin restatements composed the way VecEvalBool
composes them (oracle_select_project, tests/test_gpu_expr_program.py)."""
import numpy as np

import oracle_py as O
from test_gpu_expr_program import OracleError, oracle_select_project
from tinysql_b200.chunk import BYTES, FLOAT64, INT64, UINT64, Chunk, Column
from tinysql_b200.expression import Col, Const, Func

TP = {INT64: "int", UINT64: "uint", FLOAT64: "real"}
CMP_NAMES = ["lt", "le", "gt", "ge", "eq", "ne"]

__all__ = ["OracleError", "conds_to_program", "join_with_program"]


def conds_to_program(conds, out_types):
    """a tq_join_cond list ((op, lhs, rhs) or (op, lhs, None, const_type, value)) as the CNF filter list of comparisons"""
    filters = []
    for c in conds:
        a = Col(c[1], TP[out_types[c[1]]])
        b = Col(c[2], TP[out_types[c[2]]]) if c[2] is not None else Const(c[4], TP[c[3]])
        filters.append(Func(CMP_NAMES[c[0]], a, b))
    return filters


def _take(col, rows):
    return Column(col.tp, col.values[rows].copy(), col.not_null()[rows].copy())


def join_with_program(kind, jt, oir, inner_types, inner_cols, outer_types, outer_cols, inner_keys, outer_keys, filters, selected=None,
                      default_inner=None):
    """kind 'hash' or 'merge'.  -> (Chunk of left ++ right, division-by-zero warnings).  The rows keep the order of the oracle's
    join (the reference's order for the merge join); a miss row takes the place of its outer row's first joined row.  Raises
    OracleError with the reference's status when an evaluated joined row overflows."""
    ni, no = inner_cols[0].length, outer_cols[0].length
    it, ic = list(inner_types) + [INT64], list(inner_cols) + [Column(INT64, np.arange(ni, dtype=np.int64))]
    ot, oc = list(outer_types) + [INT64], list(outer_cols) + [Column(INT64, np.arange(no, dtype=np.int64))]
    dflt = None if default_inner is None else list(default_inner) + [None]
    if kind == "hash":
        res = O.hash_join(jt, oir, it, ic, ot, oc, inner_keys, outer_keys, selected, (), default_inner=dflt)
    else:
        res = O.merge_join(jt, oir, it, ic, ot, oc, inner_keys, outer_keys, selected, default_inner=dflt)
    n_left, n_right = (len(inner_types), len(outer_types)) if oir else (len(outer_types), len(inner_types))
    user = list(range(n_left)) + [n_left + 1 + c for c in range(n_right)]
    inner_rid, outer_rid = (n_left, n_left + 1 + n_right) if oir else (n_left + 1 + n_right, n_left)
    inner_user = set(range(n_left)) if oir else set(range(n_left, n_left + n_right))
    cols = [res.cols[i] for i in user]
    n = res.cols[0].length
    matched = res.cols[inner_rid].not_null()
    orid = res.cols[outer_rid].values
    rows = np.nonzero(matched)[0]
    passed = np.zeros(n, dtype=bool)
    warnings = 0
    if len(rows):
        _, sel, _, warnings = oracle_select_project([_take(c, rows) for c in cols], filters, [])
        passed[rows[sel.astype(bool)]] = True
    keep = ~matched | passed
    miss = np.zeros(n, dtype=bool)
    if jt != 0 and len(rows):
        survivors = np.bincount(orid[rows], weights=passed[rows], minlength=no)
        outer_ids, first = np.unique(orid[rows], return_index=True)   # the first joined row of every outer row
        miss[rows[first[survivors[outer_ids] == 0]]] = True
    keep |= miss
    out_rows = np.nonzero(keep)[0]
    out = []
    for u, c in enumerate(cols):
        vals, nn = c.values[out_rows].copy(), c.not_null()[out_rows].copy()
        if u in inner_user:
            m = miss[out_rows]
            ci = u if oir else u - n_left
            d = None if default_inner is None else default_inner[ci]
            vals[m] = (b"" if c.tp == BYTES else 0) if d is None else d
            nn[m] = d is not None
        out.append(Column(c.tp, vals, nn))
    return Chunk(out), warnings
