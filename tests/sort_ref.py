"""An exact reference for SortExec / TopNExec / MergeJoinExec over Python values, and input families aimed at the mechanics of
csrc/sort.cu (TEST INFRASTRUCTURE).

The reference does not share the kernels' or the oracle's way of comparing rows: it orders Python values (int, float, bytes,
None) with Python's own comparisons.  BIGINT and BIGINT UNSIGNED are Python ints (so -1 never equals 2^64 - 1), DOUBLE and
FLOAT are Python floats (-0.0 == 0.0, and a FLOAT cell is its exact float32 value), VARCHAR is bytes (unsigned, a proper
prefix first), NULL is first ascending and last descending (util/chunk/compare.go, executor/sort.go lessRow).  Ties keep
child order: Python's sort is stable, also with reverse=True.

`passes` restates how many radix digit passes tq_sort_stats must report: per ByItem, the key words the sort builds (the
order-preserving 64-bit words of k_sort_keys) and, per word, the 8-bit digits that are not constant over all rows.  It pins
the digit-skip mask both ways: a skipped digit that varies misorders rows, a pass over a constant digit is wasted time.

A family is a list of `Case`s; `check_family` asserts that every case has the property it is named after."""
import math
import struct
from dataclasses import dataclass, field

import numpy as np

from tinysql_b200.chunk import BYTES, FLOAT32, FLOAT64, INT64, UINT64, Column

INNER, LEFT, RIGHT = 0, 1, 2
M64 = (1 << 64) - 1
SIGN = 1 << 63
INT64_MIN, INT64_MAX, UINT64_MAX = -(1 << 63), (1 << 63) - 1, M64
SORT_MAX_BY = 8
TYPE_NAMES = {INT64: "bigint", UINT64: "ubigint", FLOAT64: "double", FLOAT32: "float", BYTES: "varchar"}
DBL_MAX, DBL_MIN, DBL_TRUE_MIN = 1.7976931348623157e308, 2.2250738585072014e-308, 5e-324
FLT_MAX, FLT_MIN, FLT_TRUE_MIN = float(np.finfo(np.float32).max), float(np.finfo(np.float32).tiny), float(np.float32(2.0 ** -149))


# ------------------------------------------------------------------------------------------------------------------ values
def f32(x):
    """the FLOAT value nearest to x, as the Python float it widens to exactly"""
    return float(np.float32(x))


def column(tp, vals, nullable=None):
    """a chunk Column of Python values (None = NULL).  nullable: give the column a NOT-NULL bitmap even without NULLs
    (None: a bitmap iff some value is NULL)"""
    has_null = any(v is None for v in vals)
    nn = [v is not None for v in vals] if (has_null or nullable) else None
    if tp == BYTES:
        return Column(BYTES, [b"" if v is None else v for v in vals], nn)
    if tp == INT64:
        raw = np.array([0 if v is None else v for v in vals], dtype=np.int64)
    elif tp == UINT64:
        raw = np.array([0 if v is None else v for v in vals], dtype=np.uint64)
    else:
        raw = np.array([0.0 if v is None else v for v in vals], dtype=np.float64 if tp == FLOAT64 else np.float32)
    return Column(tp, raw, nn)


def canon(v):
    """a value as compared for identity: floats by bit pattern (so -0.0 and 0.0 differ), the rest as they are"""
    return ("f", struct.pack("<d", v)) if isinstance(v, float) else v


def canon_rows(rows):
    return [tuple(canon(v) for v in r) for r in rows]


# ------------------------------------------------------------------------------------------------------------------ SortExec / TopN
def _key(v):
    return (0,) if v is None else (1, v)


def sort_rows(rows, by, offset=0, count=-1):
    """rows: list of tuples; by: [(column, desc)].  One stable sort per ByItem, last first; then the TopN window
    [offset, offset + count) (count < 0: all)"""
    out = list(rows)
    for col, desc in reversed(by):
        out.sort(key=lambda r: _key(r[col]), reverse=bool(desc))
    return out[offset:] if count < 0 else out[offset: offset + count]


def _enc_double(bits):
    if (bits << 1) & M64 == 0:
        return SIGN                                    # -0.0 == +0.0
    return (~bits) & M64 if bits >> 63 else bits | SIGN


def _dbits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def key_words(tp, vals, nullable):
    """the key words of one ByItem column, each a list with one word per row (before the DESC inversion)"""
    if tp == INT64:
        words = [[0 if v is None else (v & M64) ^ SIGN for v in vals]]
    elif tp == UINT64:
        words = [[0 if v is None else v for v in vals]]
    elif tp in (FLOAT64, FLOAT32):
        words = [[0 if v is None else _enc_double(_dbits(v)) for v in vals]]
    else:
        max_len = max([len(v) for v in vals if v is not None], default=0)
        words = [[0 if v is None else len(v) for v in vals]]
        for w in range((max_len + 7) // 8):
            words.append([0 if v is None else int.from_bytes(v[8 * w: 8 * w + 8].ljust(8, b"\0"), "big") for v in vals])
    if nullable:
        words.append([0 if v is None else 1 for v in vals])
    return words


def varying_digits(word_list):
    """8-bit digits of a key word that are not constant over the rows (the passes the radix sort must make)"""
    o, a = 0, M64
    for w in word_list:
        o |= w
        a &= w
    d = o ^ a
    return sum(1 for i in range(8) if (d >> (8 * i)) & 0xFF)


def passes(types, cols, nullable, by, offset=0, count=-1):
    """radix passes of tq_sort_stats: none when the input or the window is empty or there is at most one row"""
    n = len(cols[0]) if cols else 0
    lo = min(offset, n)
    m = n - lo if count < 0 else min(count, n - lo)
    if n <= 1 or m == 0:
        return 0
    total = 0
    for col, desc in by:
        for w in key_words(types[col], cols[col], nullable[col]):
            total += varying_digits([(~x) & M64 for x in w] if desc else w)
    return total


# ------------------------------------------------------------------------------------------------------------------ MergeJoinExec
def key_tuple(row, keys):
    k = tuple(row[c] for c in keys)
    return None if any(v is None for v in k) else k


def inner_sorted(irows, ik):
    """the inner rows with usable (non-NULL) keys are non-decreasing by the key tuple"""
    ks = [k for k in (key_tuple(r, ik) for r in irows) if k is not None]
    return all(a <= b for a, b in zip(ks, ks[1:]))


def merge_join(jt, outer_is_right, irows, n_inner_cols, orows, ik, ok, selected=None, default_inner=None):
    """per outer row in order: the inner rows with an equal key in inner order, or the miss row (outer joins) when there are
    none, the key has a NULL or the outer filter dropped the row; output rows = left ++ right"""
    groups = {}
    for r in irows:
        k = key_tuple(r, ik)
        if k is not None:
            groups.setdefault(k, []).append(r)
    miss = tuple(default_inner) if default_inner is not None else (None,) * n_inner_cols
    out = []
    for i, o in enumerate(orows):
        k = key_tuple(o, ok)
        hit = groups.get(k, []) if (k is not None and (selected is None or selected[i])) else []
        if not hit and jt == INNER:
            continue
        for r in (hit or [miss]):
            out.append(tuple(r) + tuple(o) if outer_is_right else tuple(o) + tuple(r))
    return out


# ------------------------------------------------------------------------------------------------------------------ families
@dataclass
class Case:
    """one input table and what runs on it.  cols: Python values per column; the last column is the row id.
    sorts: [(by, offset, count)].  A merge-join case keeps its inner table in cols / types and its outer table in ocols /
    otypes, with keys ik / ok; refused: the merge join must refuse the inner side as not sorted by its keys."""
    name: str
    types: list
    cols: list
    sorts: list = field(default_factory=list)
    nullable: list = None
    prop: object = None            # the self-check: a callable over the case
    otypes: list = None
    ocols: list = None
    ik: list = None
    ok: list = None
    onullable: list = None
    refused: bool = False

    def __post_init__(self):
        if self.nullable is None:
            self.nullable = [any(v is None for v in c) for c in self.cols]
        if self.ocols is not None and self.onullable is None:
            self.onullable = [any(v is None for v in c) for c in self.ocols]

    @property
    def n(self):
        return len(self.cols[0])

    def rows(self):
        return list(zip(*self.cols))

    def orows(self):
        return list(zip(*self.ocols))

    def columns(self):
        return [column(t, v, nb) for t, v, nb in zip(self.types, self.cols, self.nullable)]

    def ocolumns(self):
        return [column(t, v, nb) for t, v, nb in zip(self.otypes, self.ocols, self.onullable)]

    def has_float32(self):
        return FLOAT32 in self.types or FLOAT32 in (self.otypes or [])


def with_ids(name, types, cols, sorts, prop=None):
    n = len(cols[0])
    return Case(name, list(types) + [INT64], [list(c) for c in cols] + [list(range(n))], sorts, prop=prop)


def both_ways(col=0):
    return [([(col, False)], 0, -1), ([(col, True)], 0, -1)]


def _sort_passes(case, by):
    return passes(case.types, case.cols, case.nullable, by)


def digits(rng, n=600):
    """INT64 / UINT64 keys that differ in one byte only, in bit 63 only, in the lowest bit only, or not at all"""
    out = []
    for tp in (INT64, UINT64):
        base = int(rng.integers(0, 1 << 63)) | (int(rng.integers(0, 2)) << 63)
        for d in range(8):
            vals = [(base & ~(0xFF << 8 * d)) | (int(b) << 8 * d) for b in rng.integers(0, 256, n)]
            vals = [v - (1 << 64) if tp == INT64 and v >> 63 else v for v in vals]
            out.append(with_ids(f"digits_{TYPE_NAMES[tp]}_byte{d}", [tp], [vals], both_ways(),
                                lambda c, d=d: all(_sort_passes(c, by) == 1 for by, _, _ in c.sorts)
                                and len({(v & M64) >> (8 * d) & 0xFF for v in c.cols[0]}) > 1))
        if tp == INT64:
            pairs = [(-1, 0), (INT64_MIN, INT64_MAX), (5, 5 - (1 << 63))]
        else:
            pairs = [(INT64_MAX, 1 << 63), (5, 5 | SIGN), (0, UINT64_MAX)]
        vals = [pairs[int(i)][int(j)] for i, j in zip(rng.integers(0, 3, n), rng.integers(0, 2, n))]
        out.append(with_ids(f"digits_{TYPE_NAMES[tp]}_bit63", [tp], [vals], both_ways(),
                            lambda c: {5, 5 | SIGN} <= {v & M64 for v in c.cols[0]}))
        vals = [base - (1 << 64) if tp == INT64 and base >> 63 else base] * n
        out.append(with_ids(f"digits_{TYPE_NAMES[tp]}_all_equal", [tp], [vals], both_ways(), lambda c: all(_sort_passes(c, by) == 0 for by, _, _ in c.sorts)))
        lowbit = [(base & ~1) | int(b) for b in rng.integers(0, 2, n)]
        lowbit = [v - (1 << 64) if tp == INT64 and v >> 63 else v for v in lowbit]
        out.append(with_ids(f"digits_{TYPE_NAMES[tp]}_low_bit", [tp], [lowbit], both_ways(),
                            lambda c: all(_sort_passes(c, by) == 1 for by, _, _ in c.sorts) and len(set(c.cols[0])) == 2))
    return out


def _has_both_zeros(vals):
    return any(v == 0 and math.copysign(1, v) < 0 for v in vals if v is not None) and any(v == 0 and math.copysign(1, v) > 0 for v in vals if v is not None)


def _fold_matters(c):
    """sorting -0.0 strictly below +0.0 (the map without the fold) changes the row order, ASC and DESC"""
    def strict(v):
        return (0,) if v is None else (1, v, math.copysign(1, v))
    for by, _, _ in c.sorts:
        (col, desc), = by
        a = [r[-1] for r in sort_rows(c.rows(), by)]
        b = [r[-1] for r in sorted(c.rows(), key=lambda r: strict(r[col]), reverse=desc)]
        if a == b:
            return False
    return True


def _float_specials(tp):
    if tp == FLOAT64:
        one_up, one_dn = math.nextafter(1.0, math.inf), math.nextafter(1.0, -math.inf)
        big, small, tiny = DBL_MAX, DBL_MIN, DBL_TRUE_MIN
    else:
        one_up, one_dn = f32(np.nextafter(np.float32(1), np.float32(2))), f32(np.nextafter(np.float32(1), np.float32(0)))
        big, small, tiny = FLT_MAX, FLT_MIN, FLT_TRUE_MIN
    pos = [math.inf, big, small, tiny, 1.0, one_up, one_dn, 0.5, 3.0]
    return pos + [-v for v in pos] + [0.0, -0.0]


def floats(rng, tp, n=500):
    """-0.0 / +0.0 interleaved, the extremes (inf, MAX, the smallest normal and subnormal) and 1.0 / -1.0 next to their
    neighbours, as DOUBLE or as FLOAT"""
    zeros = [(-0.0 if i % 2 else 0.0) for i in range(n)]
    specials = _float_specials(tp)
    spec = [specials[int(i)] for i in rng.integers(0, len(specials), n)]
    spec_null = [None if rng.random() < 0.1 else v for v in spec]
    mixed = [v if rng.random() < 0.5 else z for v, z in zip(spec, zeros)]
    out = [with_ids(f"{TYPE_NAMES[tp]}_zeros", [tp], [zeros], both_ways(), lambda c: _has_both_zeros(c.cols[0]) and _fold_matters(c)),
           with_ids(f"{TYPE_NAMES[tp]}_zeros_and_specials", [tp], [mixed], both_ways(), lambda c: _has_both_zeros(c.cols[0]) and _fold_matters(c)),
           with_ids(f"{TYPE_NAMES[tp]}_specials", [tp], [spec_null], both_ways(),
                    lambda c: set(_float_specials(c.types[0])) <= {v for v in c.cols[0] if v is not None} and None in c.cols[0])]
    return out


def _differs_only_at(a, b, pos):
    return len(a) == len(b) and [i for i in range(len(a)) if a[i] != b[i]] == [pos]


def strings(rng):
    out = []
    pat = bytes(rng.integers(1, 256, 80, dtype=np.uint8))
    lens = [pat[:k] for k in range(73)] + [b"a" * k for k in range(73)]
    rng.shuffle(lens)
    out.append(with_ids("str_lengths_0_to_72", [BYTES], [lens], both_ways(), lambda c: {len(v) for v in c.cols[0]} == set(range(73))))
    # pairs equal but for byte 8k+7 (the last byte of a key word) or 8k+8 (the first of the next); the longest cell is 41 bytes,
    # so its differing byte sits alone in a last, partial key word
    cells, positions = [], [p for k in range(5) for p in (8 * k + 7, 8 * k + 8)]
    for pos in positions:
        base = bytes(rng.integers(1, 255, pos + 1, dtype=np.uint8))
        for delta in (-1, 1):
            cells += [base, base[:pos] + bytes([base[pos] + delta]) + base[pos + 1:]]
    out.append(with_ids("str_differ_at_8k7_8k8", [BYTES], [cells], both_ways(),
                        lambda c: max(len(v) for v in c.cols[0]) % 8 != 0
                        and all(_differs_only_at(c.cols[0][4 * j + h], c.cols[0][4 * j + h + 1], p) for j, p in enumerate(positions) for h in (0, 2))))
    nul = [b"", b"\0", b"\0\0", b"a", b"a\0", b"a\0\0", b"a\0b", b"\0a", b"a\0\0\0\0\0\0\0", b"a\0\0\0\0\0\0\0\0", b"b"]
    out.append(with_ids("str_trailing_nul", [BYTES], [[nul[int(i)] for i in rng.integers(0, len(nul), 300)]], both_ways(),
                        lambda c: {b"", b"\0", b"\0\0", b"a", b"a\0"} <= set(c.cols[0])))
    hi = [b"", b"\x7f", b"\x80", b"\xff", b"\xff\xff", b"\xff" * 8, b"\xff" * 9, b"a", b"a\x80", b"a\xff", b"\x00\xff", b"\xff\x00"]
    out.append(with_ids("str_high_bytes", [BYTES], [[hi[int(i)] for i in rng.integers(0, len(hi), 300)]], both_ways(),
                        lambda c: {b"\x80", b"\xff", b"\xff" * 8, b""} <= set(c.cols[0])))
    prefix = bytes(rng.integers(0, 256, 300, dtype=np.uint8))
    long_pre = [prefix + bytes(rng.integers(0, 3, int(rng.integers(0, 20)), dtype=np.uint8)) for _ in range(300)]
    out.append(with_ids("str_300_byte_prefix", [BYTES], [long_pre], both_ways(), lambda c: len(set(c.cols[0])) > 50))
    short = [bytes(rng.integers(0, 256, int(rng.integers(0, 12)), dtype=np.uint8)) for _ in range(400)]
    # zero bytes from byte 16 to 4998 and a 1 at the end: 625 key words, of which the 622 in the middle are constant
    short[137] = bytes(rng.integers(0, 256, 16, dtype=np.uint8)) + b"\0" * 4983 + b"\1"
    out.append(with_ids("str_one_5000_byte_cell", [BYTES], [short], both_ways(),
                        lambda c: max(len(v) for v in c.cols[0]) == 5000 and all(3 <= _sort_passes(c, by) <= 2 + 16 + 1 for by, _, _ in c.sorts)))
    en = [[b"", None, b"a", b"\0"][int(i)] for i in rng.integers(0, 4, 300)]
    out.append(with_ids("str_empty_and_null", [BYTES], [en], both_ways(), lambda c: None in c.cols[0] and b"" in c.cols[0]))
    out.append(with_ids("str_all_null", [BYTES], [[None] * 200], both_ways(), lambda c: all(v is None for v in c.cols[0])))
    out.append(with_ids("str_all_empty", [BYTES], [[b""] * 200], both_ways(),
                        lambda c: all(v == b"" for v in c.cols[0]) and all(_sort_passes(c, by) == 0 for by, _, _ in c.sorts)))
    return out


TIE_SIZES = (255, 256, 257, 4095, 4096, 4097, 3 * 4096 + 255)


def ties(rng, sizes=TIE_SIZES):
    out = []
    for n in sizes:
        k = [int(v) for v in rng.integers(-2, 3, n)]
        s = [[b"x", b"y", None][int(v)] for v in rng.integers(0, 3, n)]
        out.append(with_ids(f"ties_n{n}", [INT64, BYTES], [k, s], [([(0, False)], 0, -1), ([(1, True), (0, False)], 0, -1)],
                            lambda c: len(set(c.cols[0])) <= 5 and c.n in TIE_SIZES))
    n = 3000
    types = [INT64, UINT64, FLOAT64, FLOAT32, BYTES, INT64, UINT64, FLOAT64]
    pool = {INT64: [INT64_MIN, -1, 0, 1, INT64_MAX, None], UINT64: [0, 1, INT64_MAX, 1 << 63, UINT64_MAX, None],
            FLOAT64: [-math.inf, -1.5, -0.0, 0.0, 2.25, None], FLOAT32: [f32(-0.1), -0.0, 0.0, f32(0.1), FLT_MAX, None],
            BYTES: [b"", b"a", b"a\0", b"\xff", None]}
    cols = [[pool[t][int(i)] for i in rng.integers(0, len(pool[t]), n)] for t in types]
    by8 = [(i, bool(i % 3 == 1)) for i in (4, 0, 3, 1, 7, 2, 6, 5)]
    out.append(with_ids("ties_8_by_items", types, cols, [(by8, 0, -1), ([(i, not d) for i, d in by8], 0, -1)],
                        lambda c: len(c.sorts[0][0]) == SORT_MAX_BY and len(set(c.types[:-1])) == 5))
    out.append(with_ids("ties_same_column_asc_then_desc", [INT64, INT64], [cols[0], [int(v) for v in rng.integers(0, 3, n)]],
                        [([(0, False), (0, True), (1, True)], 0, -1), ([(1, True), (1, False), (0, False)], 0, -1)],
                        lambda c: all(by[0][0] == by[1][0] and by[0][1] != by[1][1] for by, _, _ in c.sorts)))
    return out


TOO_MANY_BY = [(0, False)] * (SORT_MAX_BY + 1)


def windows(rng, n=600):
    """TopN windows at and beyond both ends, over runs of equal keys that straddle both window edges"""
    keys = [i // 7 for i in range(n)]
    rng.shuffle(keys)
    offs = (0, 1, n - 1, n, n + 1, 1 << 62)
    cnts = (0, 1, n - 1, n, INT64_MAX)
    sorts = [([(0, False)], o, c) for o in offs for c in cnts] + [([(0, True)], 3, 10), ([(0, False)], 5, 15)]

    def straddles(c):
        ks = [r[0] for r in sort_rows(c.rows(), [(0, False)])]
        return ks[5 - 1] == ks[5] and ks[5 + 15 - 1] == ks[5 + 15]
    return [with_ids("windows", [INT64], [keys], sorts, straddles)]


def sort_families(rng):
    return digits(rng) + floats(rng, FLOAT64) + floats(rng, FLOAT32) + strings(rng) + ties(rng) + windows(rng)


# ------------------------------------------------------------------------------------------------------------------ merge-join families
def mj_case(name, itypes, icols, otypes, ocols, ik, ok, prop=None, refused=False, presort=True):
    """inner and outer tables (a row id appended to each), both sorted ascending by their keys unless presort is False"""
    ni, no = len(icols[0]), len(ocols[0])
    irows = [tuple(r) + (i,) for i, r in enumerate(zip(*icols))]
    orows = [tuple(r) + (i,) for i, r in enumerate(zip(*ocols))]
    if presort:
        irows = sort_rows(irows, [(c, False) for c in ik])
        orows = sort_rows(orows, [(c, False) for c in ok])
    icols2 = [list(c) for c in zip(*irows)] if ni else [[] for _ in range(len(icols) + 1)]
    ocols2 = [list(c) for c in zip(*orows)] if no else [[] for _ in range(len(ocols) + 1)]
    return Case(name, list(itypes) + [INT64], icols2, otypes=list(otypes) + [INT64], ocols=ocols2, ik=list(ik), ok=list(ok), prop=prop,
                refused=refused)


def mj_expect(c, jt, oir, selected=None, default_inner=None):
    return merge_join(jt, oir, c.rows(), len(c.types), c.orows(), c.ik, c.ok, selected, default_inner)


def _pairs(c):
    return len(mj_expect(c, INNER, False))


def mj_keys(rng):
    out = []
    words = [b"", b"\0", b"a", b"a\0", b"a\0\0", b"a" + b"\0" * 8, b"b", b"\xff", None]
    pick = lambda n: [words[int(i)] for i in rng.integers(0, len(words), n)]
    out.append(mj_case("mj_str_trailing_nul", [BYTES], [pick(120)], [BYTES], [pick(150)], [0], [0],
                       lambda c: b"a" in c.cols[0] and b"a\0" in c.ocols[0]
                       and all(r[0] == r[2] for r in mj_expect(c, INNER, False))))
    zi = [[-0.0, 0.0, 1.0, -1.0, None][int(i)] for i in rng.integers(0, 5, 80)]
    zo = [[0.0, -0.0, 1.0, 2.0, None][int(i)] for i in rng.integers(0, 5, 90)]
    out.append(mj_case("mj_double_zeros", [FLOAT64], [zi], [FLOAT64], [zo], [0], [0],
                       lambda c: any(math.copysign(1, r[0]) != math.copysign(1, r[2]) for r in mj_expect(c, INNER, False) if r[0] == 0)))
    fi = [[-0.0, f32(0.1), f32(-1.5), FLT_TRUE_MIN, None][int(i)] for i in rng.integers(0, 5, 80)]
    fo = [[0.0, 0.1, f32(0.1), -1.5, FLT_TRUE_MIN, 1e-46, None][int(i)] for i in rng.integers(0, 7, 100)]
    out.append(mj_case("mj_float_against_double", [FLOAT32], [fi], [FLOAT64], [fo], [0], [0],
                       lambda c: f32(0.1) != 0.1 and 0.1 in c.ocols[0] and f32(0.1) in c.cols[0]
                       and not any(r[0] == 0.1 for r in mj_expect(c, INNER, False))
                       and any(r[0] == f32(0.1) for r in mj_expect(c, INNER, False))
                       and any(r[0] == 0 and math.copysign(1, r[2]) < 0 for r in mj_expect(c, INNER, False))))
    si = [[INT64_MIN, -1, 0, 5, INT64_MAX, None][int(i)] for i in rng.integers(0, 6, 90)]
    uo = [[0, 5, INT64_MAX, 1 << 63, UINT64_MAX, None][int(i)] for i in rng.integers(0, 6, 110)]
    out.append(mj_case("mj_int_against_uint", [INT64], [si], [UINT64], [uo], [0], [0],
                       lambda c: -1 in c.cols[0] and UINT64_MAX in c.ocols[0] and 1 << 63 in c.ocols[0]
                       and {r[0] for r in mj_expect(c, INNER, False)} == {0, 5, INT64_MAX}))
    it = [INT64 if k % 2 == 0 else UINT64 for k in range(8)]
    ot = [UINT64 if t == INT64 else INT64 for t in it]
    vals = {INT64: [-1, 0, INT64_MAX], UINT64: [0, INT64_MAX, UINT64_MAX]}

    def mixed(types, n):   # mostly 0, so that all eight keys of a pair agree often; some NULLs in every column
        return [[None if rng.random() < 0.03 else (vals[t][int(rng.integers(0, 3))] if rng.random() < 0.2 else 0) for _ in range(n)] for t in types]
    out.append(mj_case("mj_eight_mixed_keys", it, mixed(it, 700), ot, mixed(ot, 700), list(range(8)), list(range(8)),
                       lambda c: len(c.ik) == 8 and all(None in col for col in c.cols[:8]) and all(None in col for col in c.ocols[:8])
                       and _pairs(c) > 0))
    si2 = [[-1, 0, 7, None][int(i)] for i in rng.integers(0, 4, 150)]
    uo2 = [[0, 7, UINT64_MAX, None][int(i)] for i in rng.integers(0, 4, 150)]
    out.append(mj_case("mj_string_and_mixed_keys", [BYTES, INT64], [pick(150), si2], [UINT64, BYTES], [uo2, pick(150)], [0, 1], [1, 0],
                       lambda c: _pairs(c) > 0 and all(r[1] == r[3] for r in mj_expect(c, INNER, False))))
    return out


def mj_unsorted(n=5000):
    """inner sides the merge join must refuse (an inversion by the key comparator) or accept"""
    out = [mj_case("mj_unsorted_nul_before_shorter", [BYTES], [[b"", b"a\0", b"a", b"b"]], [BYTES], [[b"a"]], [0], [0],
                   lambda c: not inner_sorted(c.rows(), c.ik), refused=True, presort=False)]
    first = [2, 1] + list(range(3, n + 1))
    last = list(range(1, n - 1)) + [n, n - 1]
    out.append(mj_case("mj_unsorted_first_pair", [INT64], [first], [INT64], [[1, 2, 3]], [0], [0], lambda c: not inner_sorted(c.rows(), c.ik),
                       refused=True, presort=False))
    out.append(mj_case("mj_unsorted_last_pair", [INT64], [last], [INT64], [[1, n - 1, n]], [0], [0], lambda c: not inner_sorted(c.rows(), c.ik),
                       refused=True, presort=False))
    out.append(mj_case("mj_sorted_plus_zero_before_minus_zero", [FLOAT64], [[-1.0, 0.0, -0.0, 0.0, -0.0, 2.0]], [FLOAT64], [[-0.0, 0.0, 2.0]], [0], [0],
                       lambda c: inner_sorted(c.rows(), c.ik) and _pairs(c) == 2 * 4 + 1, presort=False))
    out.append(mj_case("mj_sorted_null_between", [INT64], [[5, None, 6] * 1 + [7] * 300 + [None] * 3 + [8]], [INT64], [[5, 6, 8, None]], [0], [0],
                       lambda c: inner_sorted(c.rows(), c.ik) and not inner_sorted([r if r[0] is not None else (0, r[1]) for r in c.rows()], c.ik),
                       presort=False))
    return out


BIG_GROUPS = (4096, 16384)                         # outer rows, inner rows per outer row: 2^26 result rows
GUARD_SHAPES = {"i": (4096, (1 << 20) + 1), "ii": (8192, (1 << 19) + 1)}   # (outer rows, inner rows), all one key


def guard_total(shape):
    no, ni = GUARD_SHAPES[shape]
    return no * ni


def guard_wraps_one_tile(shape):
    """the 4096-row tiles of the scan over the outer rows' emit counts: does one tile's own sum reach 2^32?"""
    no, ni = GUARD_SHAPES[shape]
    return min(no, 4096) * ni >= 1 << 32


# ------------------------------------------------------------------------------------------------------------------ self-checks
def check_family(cases):
    for c in cases:
        assert c.prop is None or c.prop(c), f"case {c.name} does not have the property it is named after"
    return cases
