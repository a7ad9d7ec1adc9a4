"""expression.vecEval* surface (expression/builtin.go:256-263) bound to the CUDA kernels.

Each function mirrors one vectorized builtin signature: it takes evaluated argument columns and
returns the result column, raising TQError with the reference's error kinds (types.ErrOverflow…).
"""
import ctypes as C

import numpy as np

from . import _lib as L
from .chunk import BYTES, Column, FLOAT64, INT64, UINT64, VarColumn, tq_array

LT, LE, GT, GE, EQ, NE = range(6)
PLUS, MINUS, MUL, DIV = range(4)
AND, OR = 0, 1
NOT_INT, NOT_REAL, MINUS_INT, MINUS_REAL, ISNULL = range(5)
STRCMP = 6                     # tq_vec_compare_string op beyond LT..NE
STR_LENGTH, STR_ISNULL = 0, 1  # tq_vec_string_unary ops


def _u(col):
    return 1 if col.tp == UINT64 else 0


def vec_compare_int(op, a, b):
    """builtin{LT,LE,GT,GE,EQ,NE}IntSig.vecEvalInt — expression/builtin_compare_vec.go:22-292"""
    out = Column.empty(INT64, a.length)
    ta, tb, to = a.tq(), b.tq(), out.tq()
    L.check(L.load().tq_vec_compare_int(op, a.length, C.byref(ta), _u(a), C.byref(tb), _u(b), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_compare_real(op, a, b):
    """builtin{LT..NE}RealSig.vecEvalInt — expression/builtin_compare_vec_generated.go"""
    out = Column.empty(INT64, a.length)
    ta, tb, to = a.tq(), b.tq(), out.tq()
    L.check(L.load().tq_vec_compare_real(op, a.length, C.byref(ta), C.byref(tb), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_compare_string(op, a, b):
    """builtin{LT..NE}StringSig.vecEvalInt (builtin_compare_vec_generated.go:65-555); op STRCMP: builtinStrcmpSig
    (builtin_string_vec.go:52-83).  a, b: var-len columns."""
    out = Column.empty(INT64, a.length)
    ta, tb, to = a.tq(), b.tq(), out.tq()
    L.check(L.load().tq_vec_compare_string(op, a.length, C.byref(ta), C.byref(tb), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_string_unary(op, a):
    """STR_LENGTH: builtinLengthSig (builtin_string.go:75-81); STR_ISNULL: builtinStringIsNullSig (builtin_string_vec.go:21-42)"""
    out = Column.empty(INT64, a.length)
    ta, to = a.tq(), out.tq()
    L.check(L.load().tq_vec_string_unary(op, a.length, C.byref(ta), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_arith_int(op, a, b):
    """builtinArithmetic{Plus,Minus,Multiply}IntSig.vecEvalInt — expression/builtin_arithmetic_vec.go"""
    out = Column.empty(UINT64 if (_u(a) or _u(b)) else INT64, a.length)
    ta, tb, to = a.tq(), b.tq(), out.tq()
    L.check(L.load().tq_vec_arith_int(op, a.length, C.byref(ta), _u(a), C.byref(tb), _u(b), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_arith_real(op, a, b):
    """builtinArithmetic{Plus,Minus,Multiply,Divide}RealSig.vecEvalReal; returns (column, div-by-zero warnings)"""
    out = Column.empty(FLOAT64, a.length)
    ta, tb, to = a.tq(), b.tq(), out.tq()
    dz = C.c_int64(0)
    L.check(L.load().tq_vec_arith_real(op, a.length, C.byref(ta), C.byref(tb), C.byref(to), C.byref(dz), L.TQ_MEM_HOST))
    return out, dz.value


def vec_logic(op, a, b):
    """builtinLogic{And,Or}Sig.vecEvalInt — expression/builtin_op_vec.go:29-68,173-215"""
    out = Column.empty(INT64, a.length)
    ta, tb, to = a.tq(), b.tq(), out.tq()
    L.check(L.load().tq_vec_logic(op, a.length, C.byref(ta), C.byref(tb), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_unary(op, a):
    """UnaryNot / UnaryMinus / IsNull — expression/builtin_op_vec.go"""
    out_tp = FLOAT64 if op == MINUS_REAL else INT64
    out = Column.empty(out_tp, a.length)
    ta, to = a.tq(), out.tq()
    L.check(L.load().tq_vec_unary(op, a.length, C.byref(ta), _u(a), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_if(cond, a, b):
    """builtinIf{Int,Real}Sig — expression/builtin_control_vec_generated.go:117-207"""
    out = Column.empty(a.tp, a.length)
    tc, ta, tb, to = cond.tq(), a.tq(), b.tq(), out.tq()
    L.check(L.load().tq_vec_if(a.length, C.byref(tc), C.byref(ta), C.byref(tb), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_ifnull(a, b):
    """builtinIfNull{Int,Real}Sig — expression/builtin_control_vec_generated.go:23-79"""
    out = Column.empty(a.tp, a.length)
    ta, tb, to = a.tq(), b.tq(), out.tq()
    L.check(L.load().tq_vec_ifnull(a.length, C.byref(ta), C.byref(tb), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_in_int(a, lst):
    """builtinInIntSig — expression/builtin_other_vec_generated.go:24-96"""
    out = Column.empty(INT64, a.length)
    ta, to = a.tq(), out.tq()
    arr = tq_array(lst)
    flags = (C.c_int32 * max(len(lst), 1))(*[_u(c) for c in lst])
    L.check(L.load().tq_vec_in_int(a.length, C.byref(ta), _u(a), len(lst), arr, flags, C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_lt_plus_int(a, b):
    """BASELINE config 2 in one pass: (a < b, a + b) over signed BIGINT columns."""
    lt, plus = Column.empty(INT64, a.length), Column.empty(INT64, a.length)
    ta, tb, t1, t2 = a.tq(), b.tq(), lt.tq(), plus.tq()
    L.check(L.load().tq_vec_lt_plus_int(a.length, C.byref(ta), C.byref(tb), C.byref(t1), C.byref(t2), L.TQ_MEM_HOST))
    return lt, plus


def vectorized_filter(a):
    """expression.VectorizedFilter over one evaluated int column (expression/chunk_executor.go:196-245)."""
    sel = np.zeros(max(a.length, 1), dtype=np.uint8)
    ta = a.tq()
    L.check(L.load().tq_vec_filter_int(a.length, C.byref(ta), sel.ctypes.data, L.TQ_MEM_HOST))
    return sel[: a.length]


def vectorized_filter_real(a):
    """VecEvalBool / toBool for an ETReal expression (expression/expression.go:296-307): zero iff RoundFloat(f) == 0."""
    sel = np.zeros(max(a.length, 1), dtype=np.uint8)
    ta = a.tq()
    L.check(L.load().tq_vec_filter_real(a.length, C.byref(ta), sel.ctypes.data, L.TQ_MEM_HOST))
    return sel[: a.length]


def vectorized_filter_string(a):
    """VectorizedFilter over an ETString expression result: toBool = types.StrToInt(cell) != 0 (expression.go:308-322)"""
    sel = np.zeros(max(a.length, 1), dtype=np.uint8)
    ta = a.tq()
    L.check(L.load().tq_vec_filter_string(a.length, C.byref(ta), sel.ctypes.data, L.TQ_MEM_HOST))
    return sel[: a.length]


def vec_in_real(a, lst):
    """builtinInRealSig — expression/builtin_other_vec_generated.go:151-204"""
    out = Column.empty(INT64, a.length)
    ta, to = a.tq(), out.tq()
    L.check(L.load().tq_vec_in_real(a.length, C.byref(ta), len(lst), tq_array(lst), C.byref(to), L.TQ_MEM_HOST))
    return out


def vec_in_string(a, lst):
    """builtinInStringSig — expression/builtin_other_vec_generated.go:97-149"""
    out = Column.empty(INT64, a.length)
    ta, to = a.tq(), out.tq()
    L.check(L.load().tq_vec_in_string(a.length, C.byref(ta), len(lst), tq_array(lst), C.byref(to), L.TQ_MEM_HOST))
    return out


def _pick_string(fn, n, cap, *args):
    out = VarColumn.empty(BYTES, n, cap)
    to = out.tq()
    L.check(fn(n, *args, C.byref(to), L.TQ_MEM_HOST))
    return out.head(n)


def vec_if_string(cond, a, b):
    """builtinIfStringSig.vecEvalString — expression/builtin_control_vec_generated.go:209-262"""
    tc, ta, tb = cond.tq(), a.tq(), b.tq()
    return _pick_string(L.load().tq_vec_if_string, a.length, int(a.data.size + b.data.size), C.byref(tc), C.byref(ta), C.byref(tb))


def vec_ifnull_string(a, b):
    """builtinIfNullStringSig.vecEvalString — expression/builtin_control_vec_generated.go:81-112"""
    ta, tb = a.tq(), b.tq()
    return _pick_string(L.load().tq_vec_ifnull_string, a.length, int(a.data.size + b.data.size), C.byref(ta), C.byref(tb))


# ---------------------------------------------------------------------------------------------
# Fused Selection + Projection: expression trees lowered to one tq_expr_eval program
# ---------------------------------------------------------------------------------------------
X_CONST, X_CMP_INT, X_CMP_REAL, X_ARITH_INT, X_ARITH_REAL, X_LOGIC, X_UNARY, X_IF, X_IFNULL, X_FILTER, X_COMPACT = range(11)
MAX_PROGRAM_INPUTS, MAX_PROGRAM_OPS, MAX_PROGRAM_OUTPUTS = 8, 32, 4


class Expr:
    """expression.Expression (expression/expression.go:47-113) for the fixed-width builtins: a tree of Col / Const / Func
    nodes whose eval type is 'int', 'uint' (ETInt with mysql.UnsignedFlag) or 'real' (ETReal)."""
    tp = "int"


class Col(Expr):
    """expression.Column (expression/column.go): the idx-th column of the input chunk."""

    def __init__(self, idx, tp="int"):
        self.idx, self.tp = idx, tp


class Const(Expr):
    """expression.Constant (expression/constant.go); value None is NULL."""

    def __init__(self, value, tp="int"):
        self.value, self.tp = value, tp


_CMP = {"lt": LT, "le": LE, "gt": GT, "ge": GE, "eq": EQ, "ne": NE}
_ARITH = {"plus": PLUS, "minus": MINUS, "mul": MUL, "div": DIV}


class Func(Expr):
    """expression.ScalarFunction (expression/scalar_function.go) over the builtins this library implements:
    lt le gt ge eq ne | plus minus mul div | and or | not neg isnull | if ifnull | in."""

    def __init__(self, name, *args):
        self.name, self.args = name, list(args)
        real = any(a.tp == "real" for a in args)
        if name in _CMP or name in ("and", "or", "not", "isnull", "in"):
            self.tp = "int"
        elif name in _ARITH:
            self.tp = "real" if real else ("uint" if any(a.tp == "uint" for a in args) else "int")
            if name == "div" and not real:
                raise ValueError("integer division (DIV / decimal '/') is outside the vectorized builtins of the hot path")
        elif name == "neg":
            self.tp = "real" if real else "int"
        elif name == "if":
            self.tp = args[1].tp
        elif name == "ifnull":
            self.tp = args[0].tp
        else:
            raise ValueError(f"unknown builtin {name}")


class ExprProgram:
    """Lowers filters (a CNF list, expression.CNFExprs) and projection expressions to the register program of
    tq_expr_eval.  Common sub-trees are evaluated once (the reference re-evaluates them per expression)."""

    def __init__(self, n_inputs, filters=(), projections=()):
        if n_inputs > MAX_PROGRAM_INPUTS:
            raise ValueError("too many input columns for one program")
        self.n_inputs = n_inputs
        self.ops = []
        self.out_regs = []
        self.out_types = []
        self._memo = {}
        self.has_filter = bool(filters)
        for f in filters:
            r = self._lower(f)
            self._emit(X_FILTER, 1 if f.tp == "real" else 0, r)
            self._memo.clear()   # later items are evaluated on the narrowed row set; do not reuse earlier (wider) error scopes
        if filters and projections:
            self._emit(X_COMPACT, 0)
        for e in projections:
            self.out_regs.append(self._lower(e))
            self.out_types.append({"int": INT64, "uint": UINT64, "real": FLOAT64}[e.tp])
        if len(self.ops) > MAX_PROGRAM_OPS or len(self.out_regs) > MAX_PROGRAM_OUTPUTS:
            raise ValueError("expression program too long")

    def _emit(self, kind, op, a=0, b=0, c=0, ua=0, ub=0, is_null=0, imm=0):
        self.ops.append(L.TQExprOp(kind, op, a, b, c, ua, ub, is_null, imm))
        return self.n_inputs + len(self.ops) - 1

    def _key(self, e):
        if isinstance(e, Col):
            return ("c", e.idx)
        if isinstance(e, Const):
            return ("k", e.tp, e.value)
        return ("f", e.name) + tuple(self._key(a) for a in e.args)

    def _lower(self, e):
        if isinstance(e, Col):
            return e.idx
        k = self._key(e)
        if k in self._memo:
            return self._memo[k]
        if isinstance(e, Const):
            if e.value is None:
                r = self._emit(X_CONST, 0, is_null=1)
            elif e.tp == "real":
                r = self._emit(X_CONST, 0, imm=int(np.float64(e.value).view(np.uint64)))
            else:
                r = self._emit(X_CONST, 0, imm=int(e.value) & 0xFFFFFFFFFFFFFFFF)
        elif e.name == "in":
            # a IN (l0, l1, …) == (a = l0) OR (a = l1) OR …  — the same three-valued result as builtinIn{Int,Real}Sig
            acc = None
            for item in e.args[1:]:
                eq = self._lower(Func("eq", e.args[0], item))
                acc = eq if acc is None else self._emit(X_LOGIC, OR, acc, eq)
            r = acc
        else:
            regs = [self._lower(a) for a in e.args]
            tps = [a.tp for a in e.args]
            real = "real" in tps
            ua = 1 if tps[0] == "uint" else 0
            ub = 1 if len(tps) > 1 and tps[1] == "uint" else 0
            n = e.name
            if n in _CMP:
                r = self._emit(X_CMP_REAL if real else X_CMP_INT, _CMP[n], regs[0], regs[1], ua=ua, ub=ub)
            elif n in _ARITH:
                r = self._emit(X_ARITH_REAL if real else X_ARITH_INT, _ARITH[n], regs[0], regs[1], ua=ua, ub=ub)
            elif n in ("and", "or"):
                r = self._emit(X_LOGIC, AND if n == "and" else OR, regs[0], regs[1])
            elif n == "not":
                r = self._emit(X_UNARY, NOT_REAL if real else NOT_INT, regs[0])
            elif n == "neg":
                r = self._emit(X_UNARY, MINUS_REAL if real else MINUS_INT, regs[0], ua=ua)
            elif n == "isnull":
                r = self._emit(X_UNARY, ISNULL, regs[0])
            elif n == "if":
                r = self._emit(X_IF, 0, regs[0], regs[1], regs[2])
            else:
                r = self._emit(X_IFNULL, 0, regs[0], regs[1])
        self._memo[k] = r
        return r

    def run(self, cols):
        """-> (projection columns, selected uint8[n] or None, division-by-zero warnings)"""
        n = cols[0].length if cols else 0
        outs = [Column.empty(tp, n) for tp in self.out_types]
        sel = np.zeros(max(n, 1), dtype=np.uint8) if (self.has_filter or not outs) else None
        ops = (L.TQExprOp * max(len(self.ops), 1))(*self.ops)
        regs = (C.c_int32 * max(len(outs), 1))(*self.out_regs)
        dz = C.c_int64(0)
        L.check(L.load().tq_expr_eval(n, len(cols), tq_array(cols), len(self.ops), ops, len(outs), regs, tq_array(outs),
                                      sel.ctypes.data if sel is not None else None, C.byref(dz), L.TQ_MEM_HOST))
        return outs, (sel[:n] if sel is not None else None), dz.value


class JoinProgram:
    """OtherConditions of a join as the program of tq_join_set_other_program / tq_mjoin_set_other_program: filters is a CNF
    list of Expr trees over the joined row (Col(i) = output column i of left ++ right).  The referenced output columns become
    the input registers in order of first use; the trees are lowered by ExprProgram."""

    def __init__(self, filters):
        self.input_cols = []

        def remap(e):
            if isinstance(e, Col):
                if e.idx not in self.input_cols:
                    self.input_cols.append(e.idx)
                return Col(self.input_cols.index(e.idx), e.tp)
            if isinstance(e, Const):
                return e
            return Func(e.name, *[remap(a) for a in e.args])

        filters = [remap(f) for f in filters]
        self.program = ExprProgram(len(self.input_cols), filters)

    def set_on(self, setter, handle):
        """calls setter(handle, n_inputs, input_cols, n_ops, ops) and checks its status"""
        cols = (C.c_int32 * max(len(self.input_cols), 1))(*self.input_cols)
        ops = (L.TQExprOp * max(len(self.program.ops), 1))(*self.program.ops)
        L.check(setter(handle, len(self.input_cols), cols, len(self.program.ops), ops))
