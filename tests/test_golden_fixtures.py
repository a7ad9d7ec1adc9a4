"""The reference's own known-answer cases (tests/golden/reference_cases.json, transcribed from the Go test-suite by
tests/golden/make_golden.py with file:line citations) run against BOTH engines:
  * the CPU oracle (`-m "not gpu"`): this is what pins the oracle to the reference;
  * the CUDA path through the C-ABI (`-m gpu`): HashJoinExec / HashAggExec / vecEval* on the same cases."""
import json
import os

import numpy as np
import pytest

import oracle_py as O
from tinysql_b200.chunk import BYTES, FLOAT32, FLOAT64, INT64, UINT64, Chunk, Column

CASES = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_cases.json")))
TP = {"int64": INT64, "uint64": UINT64, "float64": FLOAT64, "bytes": BYTES, "float32": FLOAT32}
NP = {INT64: np.int64, UINT64: np.uint64, FLOAT64: np.float64, FLOAT32: np.float32}
JT = {"inner": 0, "left": 1, "right": 2}
FN = {"count": 0, "sum": 1, "avg": 2, "max": 3, "min": 4, "firstrow": 5}


def col(tp, vals):
    if tp == BYTES:
        return Column(BYTES, [None if v is None else v.encode("utf-8") for v in vals])
    return Column(tp, np.array([0 if v is None else v for v in vals], dtype=NP[tp]), [v is not None for v in vals])


def table(rows, ncols, types=None):
    types = types or [INT64] * ncols
    return [col(types[c], [r[c] for r in rows]) for c in range(ncols)]


# ------------------------------------------------------------------ engines
class OracleEngine:
    name = "oracle"

    def join(self, jt, outer_is_right, btypes, bcols, ptypes, pcols, bkeys, pkeys, selected, limit):
        rows = O.hash_join(jt, outer_is_right, btypes, bcols, ptypes, pcols, bkeys, pkeys, selected).rows()
        return rows[:limit] if limit else rows  # the Limit above the join stops pulling after `limit` rows

    def agg(self, types, cols, group_by, funcs, workers):
        rc, out = O.hash_agg(types, cols, group_by, funcs, workers)
        assert rc == 0
        return out.rows()

    def arith(self, op, a, b):
        if a.tp == FLOAT64:
            rc, out, _ = O.vec_arith_real(op, a, b)
        else:
            rc, out = O.vec_arith_int(op, a, b)
        assert rc == 0
        return out

    def compare(self, op, a, b):
        if a.tp == BYTES:
            rc, out = O.vec_compare_string(op, a, b)
        else:
            rc, out = O.vec_compare_real(op, a, b) if a.tp == FLOAT64 else O.vec_compare_int(op, a, b)
        assert rc == 0
        return out

    def length(self, a):
        rc, out = O.vec_string_unary(0, a)
        assert rc == 0
        return out

    def unary(self, op, a):
        rc, out = O.vec_unary(op, a)
        assert rc == 0
        return out

    def in_int(self, a, lst):
        rc, out = O.vec_in_int(a, lst)
        assert rc == 0
        return out


class GpuEngine:
    name = "gpu"

    def join(self, jt, outer_is_right, btypes, bcols, ptypes, pcols, bkeys, pkeys, selected, limit):
        from tinysql_b200.executor import HashJoinExec, MockDataSource
        inner, outer = MockDataSource(btypes, bcols), MockDataSource(ptypes, pcols)
        filt = (lambda chk: selected[: chk.num_rows()]) if selected is not None else None  # every case fits one chunk
        e = HashJoinExec(outer, inner, pkeys, bkeys, jt, outer_is_right, filt)
        e.Open()
        if limit:  # `limit N` then Close while the join still has rows to give (join_test.go:175-182)
            got = e.Next(limit)
        else:
            got = e.drain()
        e.Close()
        return got.rows()

    def agg(self, types, cols, group_by, funcs, workers):
        from tinysql_b200.executor import HashAggExec, MockDataSource
        e = HashAggExec(MockDataSource(types, cols), group_by, funcs)
        e.Open()
        got = e.drain()
        e.Close()
        return got.rows()

    def arith(self, op, a, b):
        from tinysql_b200 import expression as E
        return E.vec_arith_real(op, a, b)[0] if a.tp == FLOAT64 else E.vec_arith_int(op, a, b)

    def compare(self, op, a, b):
        from tinysql_b200 import expression as E
        if a.tp == BYTES:
            return E.vec_compare_string(op, a, b)
        return E.vec_compare_real(op, a, b) if a.tp == FLOAT64 else E.vec_compare_int(op, a, b)

    def length(self, a):
        from tinysql_b200 import expression as E
        return E.vec_string_unary(E.STR_LENGTH, a)

    def unary(self, op, a):
        from tinysql_b200 import expression as E
        return E.vec_unary(op, a)

    def in_int(self, a, lst):
        from tinysql_b200 import expression as E
        return E.vec_in_int(a, lst)


ENGINES = [pytest.param(OracleEngine(), id="oracle"), pytest.param(GpuEngine(), id="gpu", marks=pytest.mark.gpu)]


@pytest.fixture
def engine(request):
    eng = request.param
    if eng.name == "gpu":
        request.getfixturevalue("lib")  # loads libtinysql_b200.so and needs an H100
    return eng


def key(r):
    return tuple((0, 0) if v is None else (1, str(v)) for v in r)


def norm(v):
    """cells as the golden file spells them: strings for var-len cells, FLOAT values rounded through float32"""
    if isinstance(v, bytes):
        return v.decode("utf-8")
    if isinstance(v, float):
        return float(np.float32(v))
    return v


# ------------------------------------------------------------------ joins
def run_join_case(eng, case, build):
    lhs, rhs = case["lhs"], case["rhs"]
    ncl, ncr = len(lhs[0]), len(rhs[0])
    lt = [TP[t] for t in case["ltypes"]] if "ltypes" in case else [INT64] * ncl
    rt = [TP[t] for t in case["rtypes"]] if "rtypes" in case else [INT64] * ncr
    l, r = table(lhs, ncl, lt), table(rhs, ncr, rt)
    jt = JT[case["type"]]
    if build == "rhs":      # probe (outer) side is the left child
        rows = eng.join(jt, False, rt, r, lt, l, case["rkey"], case["lkey"], _sel(case), case.get("limit"))
    else:
        rows = eng.join(jt, True, lt, l, rt, r, case["lkey"], case["rkey"], _sel(case), case.get("limit"))
    if "where" in case:
        rows = [x for x in rows if eval(case["where"], {}, {"r": x})]
    if "select" in case:
        rows = [tuple(x[c] for c in case["select"]) for x in rows]
    return rows


def _sel(case):
    return np.array(case["outer_selected"], dtype=np.uint8) if "outer_selected" in case else None


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
@pytest.mark.parametrize("case", CASES["join"], ids=lambda c: c["name"])
def test_reference_join_goldens(engine, case):
    # outer joins build on the non-outer side (builder.go:451-477); inner joins must give the same rows either way
    builds = {"left": ["rhs"], "right": ["lhs"], "inner": [case["build"]] if "build" in case else ["rhs", "lhs"]}[case["type"]]
    for build in builds:
        rows = [tuple(norm(v) for v in x) for x in run_join_case(engine, case, build)]
        want = [tuple(norm(v) for v in x) for x in case["expect"]]
        if case.get("ordered"):
            assert rows == want, (case["cite"], build)
        else:
            assert sorted(rows, key=key) == sorted(want, key=key), (case["cite"], build)


# ------------------------------------------------------------------ aggregation
@pytest.mark.parametrize("engine", ENGINES, indirect=True)
@pytest.mark.parametrize("case", CASES["agg"], ids=lambda c: c["name"])
def test_reference_agg_goldens(engine, case):
    types = [TP[t] for t, _ in case["cols"]]
    cols = [col(TP[t], v) for t, v in case["cols"]]
    funcs = [(FN[f], a) for f, a in case["funcs"]]
    rows = engine.agg(types, cols, case["group_by"], funcs, case.get("partial_workers", 1))
    want = [tuple(x) for x in case["expect"]]
    assert sorted(rows, key=key) == sorted(want, key=key), case["cite"]


# ------------------------------------------------------------------ vectorized builtins
ARITH = {"plus": 0, "minus": 1, "mul": 2}
CMP = {"lt": 0, "le": 1, "gt": 2, "ge": 3, "eq": 4, "ne": 5, "strcmp": 6}


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
@pytest.mark.parametrize("case", CASES["expr"], ids=lambda c: c["op"] + "@" + c["cite"].split(":")[-1])
def test_reference_builtin_goldens(engine, case):
    from tinysql_b200 import expression as E
    assert (E.PLUS, E.MINUS, E.MUL) == (0, 1, 2) and (E.LT, E.EQ) == (CMP["lt"], CMP["eq"])
    args = [col(TP[t], [v]) for t, v in case["args"]]
    if case["op"] in ARITH:
        out = engine.arith(ARITH[case["op"]], args[0], args[1])
    elif case["op"] in CMP:
        out = engine.compare(CMP[case["op"]], args[0], args[1])
    elif case["op"] == "length":
        out = engine.length(args[0])
    elif case["op"] == "neg":
        out = engine.unary(E.MINUS_REAL if args[0].tp == FLOAT64 else E.MINUS_INT, args[0])
    elif case["op"] == "isnull":
        out = engine.unary(E.ISNULL, args[0])
    else:
        out = engine.in_int(args[0], args[1:])
    tp, want = TP[case["expect"][0]], case["expect"][1]
    assert out.tp == tp or want is None
    got = out.tolist()[0]
    if want is None:
        assert got is None, case["cite"]
    else:
        assert got == NP[tp](want), case["cite"]


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
@pytest.mark.parametrize("case", CASES["key_equality"], ids=lambda c: c["cite"].split(":")[-1])
def test_reference_key_equality_goldens(engine, case):
    (ta, va), (tb, vb) = case["a"], case["b"]
    rows = engine.join(0, False, [TP[ta]], [col(TP[ta], [va])], [TP[tb]], [col(TP[tb], [vb])], [0], [0], None, None)
    assert (len(rows) == 1) == case["equal"], case["cite"]
