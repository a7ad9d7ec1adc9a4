"""Operands at the overflow and sign boundaries of the fixed-width builtins (TEST INFRASTRUCTURE).

Pools of BIGINT, BIGINT UNSIGNED and DOUBLE values around every limit a check of the reference tests, and pair generators aimed
at the limits of each operation: sums and differences at `limit - y + {-1, 0, 1}`, products at `limit / y + {-1, 0, 1}` for y
of every magnitude and sign, double sums that land exactly on DBL_MAX, one ulp past it, or round back to it.  Values are
Python numbers of the operand's SQL type (see vec_statements.py); columns() builds the chunk columns with NULL rows whose
slots hold edge values too."""
import math

import numpy as np

from tinysql_b200.chunk import FLOAT64, INT64, UINT64, Column
from vec_statements import DBL_MAX, I64_MAX, I64_MIN, U64_MAX

INT64_POOL = sorted({0, 1, -1, 2, -2,
                     (1 << 31) + 1, (1 << 31) - 1, -(1 << 31) - 1, -(1 << 31) + 1,
                     (1 << 32) + 1, (1 << 32) - 1, -(1 << 32) - 1, -(1 << 32) + 1,
                     (1 << 62) + 1, (1 << 62) - 1, -(1 << 62) - 1, -(1 << 62) + 1,
                     I64_MAX, I64_MAX - 1, I64_MIN, I64_MIN + 1})
UINT64_POOL = sorted({0, 1, 2, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, U64_MAX - 1, U64_MAX})

_HALF_DOWN, _HALF_UP = math.nextafter(0.5, 0), math.nextafter(0.5, 1)   # 0.49999999999999994, 0.5000000000000001
_SQRT_MAX = math.sqrt(DBL_MAX)
FLOAT64_POOL = sorted({s * v for s in (1.0, -1.0) for v in (
    0.0, 5e-324, 2.2250738585072014e-308, 0.5, _HALF_DOWN, _HALF_UP, 1.0, 1.5, 2.0,
    1e154, math.nextafter(1e154, 0), math.nextafter(1e154, math.inf),
    _SQRT_MAX, math.nextafter(_SQRT_MAX, 0), math.nextafter(_SQRT_MAX, math.inf),
    DBL_MAX, DBL_MAX / 2, math.nextafter(DBL_MAX, 0))}, key=lambda v: (v, math.copysign(1, v)))
# toBool and the comparisons also meet the non-finite values
FLOAT64_FILTER_POOL = FLOAT64_POOL + [math.inf, -math.inf, math.nan]

INT_MIXES = [(False, False), (True, True), (True, False), (False, True)]   # (a unsigned, b unsigned)


def pool(unsigned):
    return UINT64_POOL if unsigned else INT64_POOL


def _fits(v, unsigned):
    return 0 <= v <= U64_MAX if unsigned else I64_MIN <= v <= I64_MAX


def _magnitudes(rng, unsigned, k=3):
    """random operands of every magnitude 2^0 .. 2^63, both signs where the type has them"""
    out = []
    for e in range(64):
        for _ in range(k):
            v = int(rng.integers(1 << max(e - 1, 0), 1 << e, dtype=np.uint64, endpoint=True)) if e else 1
            if not unsigned and rng.random() < 0.5:
                v = -v
            if _fits(v, unsigned):
                out.append(v)
    return out


def int_pairs(op, ua, ub, seed=0):
    """-> [(x, y)]: the cross product of the pools plus pairs aimed at the limits of op (0 plus, 1 minus, 2 mul) for this
    sign mix; both operands in their types' ranges, no duplicates"""
    rng = np.random.default_rng(seed * 131 + op * 7 + 2 * ua + ub)
    pairs = {(x, y) for x in pool(ua) for y in pool(ub)}
    limits = (0, U64_MAX, I64_MIN, I64_MAX, 1 << 63)
    ys = pool(ub) + _magnitudes(rng, ub)
    xs = pool(ua) + _magnitudes(rng, ua)
    for lim in limits:
        for d in (-1, 0, 1):
            for y in ys:
                if op == 0:
                    x = lim - y + d           # x + y == lim + d
                elif op == 1:
                    x = lim + y + d           # x - y == lim + d
                else:
                    if y == 0:
                        continue
                    x = lim // y + d
                if _fits(x, ua):
                    pairs.add((x, y))
            for x in xs:                      # and y aimed for a given x
                if op == 0:
                    y = lim - x + d
                elif op == 1:
                    y = x - lim + d
                else:
                    if x == 0:
                        continue
                    y = lim // x + d
                if _fits(y, ub):
                    pairs.add((x, y))
    return sorted(pairs)


def real_pairs(op, seed=0):
    """-> [(x, y)] over the DOUBLE pool plus pairs aimed at DBL_MAX: x + y exactly DBL_MAX, one ulp past it, sums the
    reference's `y > MaxFloat64 - x` check and isinf(x + y) judge differently; products and quotients at DBL_MAX / y"""
    rng = np.random.default_rng(seed * 17 + op)
    pairs = {(x, y) for x in FLOAT64_POOL for y in FLOAT64_POOL}
    xs = FLOAT64_POOL + [float(v) for v in rng.uniform(-1, 1, 40) * DBL_MAX] + [DBL_MAX * 0.75, 1e308, 8e307]
    for x in xs:
        for s in (1.0, -1.0):
            if op in (0, 1):
                y0 = s * DBL_MAX - x if op == 0 else x - s * DBL_MAX       # the rounded remainder the check compares with
                cands = [y0, math.nextafter(y0, math.inf), math.nextafter(y0, -math.inf)]
                cands += [y0 + math.copysign(u, y0) for u in (1.0, 2.0 ** 969, 2.0 ** 970, 2.0 ** 971)]
            else:
                if x == 0:
                    continue
                y0 = s * DBL_MAX / x if op == 2 else x / (s * DBL_MAX)
                cands = [y0, math.nextafter(y0, math.inf), math.nextafter(y0, -math.inf)]
            for y in cands:
                if math.isfinite(y):
                    pairs.add((x, y))
    # DBL_MAX + tiny: finite sum that the check still rejects
    for t in (1.0, 2.0 ** 969, 2.0 ** 970, math.nextafter(2.0 ** 970, 0), 1e292):
        pairs.update({(DBL_MAX, t), (t, DBL_MAX), (-DBL_MAX, -t), (-t, -DBL_MAX), (DBL_MAX, -t), (-DBL_MAX, t)})
    return sorted(pairs, key=lambda p: (p[0], math.copysign(1, p[0]), p[1], math.copysign(1, p[1])))


def np_values(vals, tp):
    if tp == FLOAT64:
        return np.array(vals, dtype=np.float64)
    if tp == UINT64:
        return np.array(vals, dtype=np.uint64)
    return np.array(vals, dtype=np.int64)


def column(vals, tp, not_null=None):
    return Column(tp, np_values(vals, tp), not_null)


def null_mask(rng, n, frac=0.2):
    return rng.random(n) >= frac
