"""The key-less hash join (no key columns) for the parity tests (TEST INFRASTRUCTURE).

With no key columns hashRowContainer.PutChunk hashes nothing: every build row gets the FNV offset basis and goes into ONE
chain, in insertion order (executor/hash_table.go:146-169), and every selected probe row finds that chain with matchJoinKey
true over zero columns (join.go:325-362, rowHashMap.Get hash_table.go:259-272).  The oracle's hash join has exactly that
shape when both sides carry one constant NOT NULL key column, so keyless_hash_join / keyless_join_with_program append one,
join on it with the oracle's chain code and drop it again.

nested_loop is an independent restatement in numpy: np.repeat of the probe rows x np.tile of the build rows, masks for
`selected` and for the conditions, the miss row of an outer probe row placed at that probe row.
"""
import numpy as np

import oracle_py as O
from join_program_oracle import join_with_program
from tinysql_b200.chunk import BYTES, INT64, Chunk, Column
from tinysql_b200.expression import Col, Const, Func


def _key(n):
    return Column(INT64, np.zeros(n, dtype=np.int64))


def _shift(u, n_left):
    return u if u < n_left else u + 1


def _drop(chunk, n_left):
    cols = chunk.cols
    return Chunk(cols[:n_left] + cols[n_left + 1:-1])


def keyless_hash_join(jt, oir, build_types, build_cols, probe_types, probe_cols, selected=None, conds=(), default_inner=None):
    """O.hash_join with no key columns.  conds / default_inner as for O.hash_join, over the output row left ++ right."""
    n_left = len(build_types) if oir else len(probe_types)
    sc = [tuple([c[0], _shift(c[1], n_left), None if c[2] is None else _shift(c[2], n_left)] + list(c[3:])) for c in conds]
    dflt = None if default_inner is None else list(default_inner) + [None]
    res = O.hash_join(jt, oir, list(build_types) + [INT64], list(build_cols) + [_key(build_cols[0].length)], list(probe_types) + [INT64],
                      list(probe_cols) + [_key(probe_cols[0].length)], [len(build_types)], [len(probe_types)], selected, sc, dflt)
    return _drop(res, n_left)


def _shift_expr(e, n_left):
    if isinstance(e, Col):
        return Col(_shift(e.idx, n_left), e.tp)
    if isinstance(e, Const):
        return e
    return Func(e.name, *[_shift_expr(a, n_left) for a in e.args])


def keyless_join_with_program(jt, oir, inner_types, inner_cols, outer_types, outer_cols, filters, selected=None, default_inner=None):
    """join_with_program('hash', ...) with no key columns -> (Chunk, division-by-zero warnings); raises OracleError"""
    n_left = len(inner_types) if oir else len(outer_types)
    dflt = None if default_inner is None else list(default_inner) + [None]
    res, warn = join_with_program("hash", jt, oir, list(inner_types) + [INT64], list(inner_cols) + [_key(inner_cols[0].length)],
                                  list(outer_types) + [INT64], list(outer_cols) + [_key(outer_cols[0].length)], [len(inner_types)],
                                  [len(outer_types)], [_shift_expr(f, n_left) for f in filters], selected, dflt)
    return _drop(res, n_left), warn


def _gather(col, idx, miss, default=None):
    """col's rows idx; rows where miss is set take `default` (None = NULL)"""
    safe = np.where(miss, 0, idx)
    nn = col.not_null()[safe] & ~miss if col.length else np.zeros(len(idx), dtype=bool)
    if col.tp == BYTES:
        cells = col.values if col.length else []
        return Column(BYTES, [cells[i] if ok else None for i, ok in zip(safe, nn)], nn)
    vals = col.values[safe].copy() if col.length else np.zeros(len(idx), dtype=col.values.dtype)
    if default is not None:
        vals[miss] = default
        nn = nn | miss
    return Column(col.tp, vals, nn)


def nested_loop(jt, oir, build_cols, probe_cols, selected=None, passes=None, default_inner=None):
    """The key-less join in numpy.  passes(pi, bi) -> bool array: the conditions of the pairs (probe row pi, build row bi)."""
    nb, npr = build_cols[0].length, probe_cols[0].length
    pi = np.repeat(np.arange(npr), nb)
    bi = np.tile(np.arange(nb), npr)
    keep = np.ones(len(pi), dtype=bool) if selected is None else np.asarray(selected, dtype=bool)[pi]
    if passes is not None and len(pi):
        keep &= np.asarray(passes(pi, bi), dtype=bool)
    out_p, out_b = pi[keep], bi[keep]
    if jt != 0:
        survivors = np.bincount(out_p, minlength=npr)
        lone = np.nonzero(survivors == 0)[0]
        out_p = np.concatenate([out_p, lone])
        out_b = np.concatenate([out_b, np.full(len(lone), -1)])
        order = np.argsort(out_p, kind="stable")
        out_p, out_b = out_p[order], out_b[order]
    miss = out_b < 0
    pcols = [_gather(c, out_p, np.zeros(len(out_p), dtype=bool)) for c in probe_cols]
    bcols = [_gather(c, out_b, miss, None if default_inner is None else default_inner[k]) for k, c in enumerate(build_cols)]
    return Chunk(bcols + pcols if oir else pcols + bcols)
