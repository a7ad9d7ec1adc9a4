"""The per-row statements of the reference's vectorized fixed-width builtins, restated in Python (TEST INFRASTRUCTURE).

Written from the Go sources, independently of oracle/oracle.c: expression/builtin_arithmetic_vec.go (plus / minus / multiply /
divide), builtin_op_vec.go (unary minus), types/compare.go (VecCompare*, CompareFloat64), builtin_compare_vec.go (vecResOf*),
expression.go (toBool), types/helper.go (RoundFloat), builtin_other_vec_generated.go (IN).  Go's int64 / uint64 arithmetic
wraps, so every statement goes through the explicit 64-bit helpers i64() / u64() and go_div() (truncating, MinInt64 / -1 ==
MinInt64); Python floats are IEEE doubles, so the real statements are exact.

An integer operand is given as the value of its SQL type (a Python int in [-2^63, 2^63) for BIGINT, [0, 2^64) for BIGINT
UNSIGNED); Go holds both as int64 (`lhi64s[i]`).  Every function covers one non-NULL row and returns
(value, error kind or None, branch tag): the value is the 64-bit pattern of the result (None where the statement returns the
error or the row becomes NULL); the error kind is the status the library reports (TQ_ERR_OVERFLOW_*); the tag names the Go
`if` that decided the row, as `function:line`.
"""
import math

I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1
BIGINT, UBIGINT, DOUBLE = 3, 4, 5           # TQ_ERR_OVERFLOW_BIGINT / _BIGINT_UNSIGNED / _DOUBLE
DBL_MAX = 1.7976931348623157e308            # math.MaxFloat64
PLUS, MINUS, MUL, DIV = range(4)


def u64(x):
    """uint64(x): the two's-complement pattern"""
    return x & U64_MAX


def i64(x):
    """int64(x): wraps like Go's int64 arithmetic"""
    x &= U64_MAX
    return x - (1 << 64) if x >> 63 else x


def go_div(a, b):
    """Go's int64 a / b (b != 0): truncates toward zero, MinInt64 / -1 wraps to MinInt64"""
    q = abs(a) // abs(b)
    return i64(q if (a < 0) == (b < 0) else -q)


def _int_result(v):
    return u64(v), None, None


# ------------------------------------------------------------------ builtinArithmeticPlusIntSig  builtin_arithmetic_vec.go:428-495
def plus_int(x, y, ua, ub):
    lh, rh = i64(x), i64(y)
    if ua and ub:                                                            # plusUU
        if u64(lh) > U64_MAX - u64(rh):
            return None, UBIGINT, "plusUU:435"
    elif ua:                                                                 # plusUS (tests lh twice)
        if rh < 0 and u64(i64(-rh)) > u64(lh):
            return None, UBIGINT, "plusUS:451"
        if rh > 0 and u64(lh) > U64_MAX - u64(lh):
            return None, UBIGINT, "plusUS:454"
    elif ub:                                                                 # plusSU
        if lh < 0 and u64(i64(-lh)) > u64(rh):
            return None, UBIGINT, "plusSU:470"
        if lh > 0 and u64(rh) > U64_MAX - u64(lh):
            return None, UBIGINT, "plusSU:473"
    else:                                                                    # plusSS
        if lh > 0 and rh > I64_MAX - lh:
            return None, BIGINT, "plusSS:488 lh>0"
        if lh < 0 and rh < I64_MIN - lh:
            return None, BIGINT, "plusSS:488 lh<0"
    return _int_result(lh + rh)


# ------------------------------------------------------------------ builtinArithmeticMinusIntSig  :205-269 (forceToSigned off)
def minus_int(x, y, ua, ub):
    lh, rh = i64(x), i64(y)
    if ua and ub:                                                            # minusUU
        if u64(lh) < u64(rh):
            return None, UBIGINT, "minusUU:212"
    elif ua:                                                                 # minusUS
        if rh >= 0 and u64(lh) < u64(rh):
            return None, UBIGINT, "minusUS:228"
        if rh < 0 and u64(lh) > U64_MAX - u64(i64(-rh)):
            return None, UBIGINT, "minusUS:231"
    elif ub:                                                                 # minusSU: lh - MinInt64 wraps
        if u64(i64(lh - I64_MIN)) < u64(rh):
            return None, UBIGINT, "minusSU:247"
    else:                                                                    # minusSS: -rh wraps
        if lh > 0 and i64(-rh) > I64_MAX - lh:
            return None, BIGINT, "minusSS:262 lh>0"
        if lh < 0 and i64(-rh) < I64_MIN - lh:
            return None, BIGINT, "minusSS:262 lh<0"
    return _int_result(lh - rh)


# ------------------------------------------------------------------ multiply: builtin_arithmetic.go:344-348 picks
# MultiplyIntUnsigned when either operand is unsigned
def mul_int(x, y, ua, ub):
    if ua or ub:                                                             # MultiplyIntUnsigned :516-531
        a, b = u64(x), u64(y)
        res = u64(a * b)
        if a != 0 and res // a != b:
            return None, UBIGINT, "MultiplyIntUnsigned:526"
        return _int_result(res)
    a, b = i64(x), i64(y)                                                    # MultiplyInt :323-339
    tmp = i64(a * b)
    if a != 0 and go_div(tmp, a) != b:
        return None, BIGINT, "MultiplyInt:333"
    return _int_result(tmp)


ARITH_INT = {PLUS: plus_int, MINUS: minus_int, MUL: mul_int}


def arith_int(op, x, y, ua, ub):
    return ARITH_INT[op](x, y, ua, ub)


# ------------------------------------------------------------------ builtinUnaryMinusIntSig  builtin_op_vec.go:221-243
def neg_int(x, ua):
    """The Go loops have no NULL test; NULL slots are don't-care in the column contract, so callers skip NULL rows."""
    v = i64(x)
    if ua:
        if u64(v) > (1 << 63):                                               # uint64(-math.MinInt64) == 2^63
            return None, BIGINT, "UnaryMinusInt:229"
    elif v == I64_MIN:
        return None, BIGINT, "UnaryMinusInt:236"
    return _int_result(-v)


# ------------------------------------------------------------------ real arithmetic  builtin_arithmetic_vec.go
def plus_real(x, y):                                                         # builtinArithmeticPlusRealSig :292-300
    if x > 0 and y > DBL_MAX - x:
        return None, DOUBLE, "PlusReal:296 x>0"
    if x < 0 and y < -DBL_MAX - x:
        return None, DOUBLE, "PlusReal:296 x<0"
    return x + y, None, None


def minus_real(x, y):                                                        # builtinArithmeticMinusRealSig :79-87
    if x > 0 and -y > DBL_MAX - x:
        return None, DOUBLE, "MinusReal:83 x>0"
    if x < 0 and -y < -DBL_MAX - x:
        return None, DOUBLE, "MinusReal:83 x<0"
    return x - y, None, None


def mul_real(x, y):                                                          # builtinArithmeticMultiplyRealSig :46-54
    r = x * y
    if math.isinf(r):
        return None, DOUBLE, "MultiplyReal:51"
    return r, None, None


def div_real(x, y):                                                          # builtinArithmeticDivideRealSig :365-381
    if y == 0:                                                               # handleDivisionByZeroError: a warning, the row is NULL
        return None, None, "DivideReal:369"
    r = x / y
    if math.isinf(r):
        return None, DOUBLE, "DivideReal:378"
    return r, None, None


ARITH_REAL = {PLUS: plus_real, MINUS: minus_real, MUL: mul_real, DIV: div_real}


def arith_real(op, x, y):
    return ARITH_REAL[op](x, y)


# ------------------------------------------------------------------ comparisons
def compare_int(x, y, ua, ub):
    """types.VecCompare{UU,II,UI,IU} (types/compare.go:44-101) -> (-1 / 0 / 1, tag)"""
    if ua and ub:
        a, b = u64(x), u64(y)
        return (-1 if a < b else (0 if a == b else 1)), "VecCompareUU"
    if not ua and not ub:
        a, b = i64(x), i64(y)
        return (-1 if a < b else (0 if a == b else 1)), "VecCompareII"
    if ua:
        a, b = u64(x), i64(y)
        if b < 0 or a > I64_MAX:
            return 1, "VecCompareUI:75"
        a = i64(a)
        return (-1 if a < b else (0 if a == b else 1)), "VecCompareUI:77"
    a, b = i64(x), u64(y)
    if a < 0 or b > I64_MAX:
        return -1, "VecCompareIU:91"
    b = i64(b)
    return (-1 if a < b else (0 if a == b else 1)), "VecCompareIU:93"


def compare_float(x, y):
    """types.CompareFloat64 (types/compare.go:104-112): NaN compares as 1"""
    return -1 if x < y else (0 if x == y else 1)


CMP_RES = [lambda c: c < 0, lambda c: c <= 0, lambda c: c > 0, lambda c: c >= 0, lambda c: c == 0, lambda c: c != 0]   # vecResOf{LT..NE}


def cmp_result(op, c):
    """builtin_compare_vec.go:214-279"""
    return int(CMP_RES[op](c))


# ------------------------------------------------------------------ toBool  expression.go:281-309
def round_float(f):
    """types.RoundFloat (types/helper.go:28-34): round half away from zero"""
    if abs(f) < 0.5:
        return 0.0
    return float(math.trunc(f + math.copysign(0.5, f))) if math.isfinite(f) else f + math.copysign(0.5, f)


def to_bool_int(v):
    """1 / 0 for a non-NULL ETInt row: i64s[i] == 0 is zero"""
    return int(v != 0)


def to_bool_real(f):
    """1 / 0 for a non-NULL ETReal row: RoundFloat(f) == 0 is zero (NaN rounds to NaN, which is not zero)"""
    return int(not (round_float(f) == 0))


# ------------------------------------------------------------------ builtinInIntSig  builtin_other_vec_generated.go:24-90
def in_int(x, ua, items):
    """items: [(value or None for NULL, unsigned)]; x is not NULL.  -> 1, 0 or None (NULL)"""
    has_null = False
    for y, u in items:
        if y is None:
            has_null = True
            continue
        a0, a1 = i64(x), i64(y)
        if ua == u:
            eq = a1 == a0
        elif not ua:
            eq = a0 >= 0 and a1 == a0
        else:
            eq = a1 >= 0 and a1 == a0
        if eq:
            return 1
    return None if has_null else 0
