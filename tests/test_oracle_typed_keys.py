"""CPU suite: the oracle's restatement of FLOAT / var-len key encoding, string GROUP BY and string / FLOAT aggregate
arguments, pinned against the reference's own known answers (paths relative to the reference repository) and against an independent
pure-Python restatement."""
import ctypes as C
from collections import defaultdict

import numpy as np
import pytest

import oracle_py as O
from test_oracle_golden import _hash, fnv1_64
from tinysql_b200.chunk import BYTES, FLOAT32, FLOAT64, INT64, UINT64, Chunk, Column, tq_array

COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)


def _equal(t1, c1, r1, t2, c2, r2):
    return O.load().orc_equal_row(C.c_int(1), (C.c_int * 1)(t1), tq_array([c1]), (C.c_int * 1)(0), C.c_int64(r1),
                                  (C.c_int * 1)(t2), tq_array([c2]), (C.c_int * 1)(0), C.c_int64(r2))


def test_hash_chunk_row_float_and_bytes_equalities():
    # util/codec/codec_test.go:764-768 TestHashChunkRow: float32(1.0) == float64(1.0), != float64(1.1); "x" == []byte("x"), != "y"
    f32, f64 = Column(FLOAT32, [1.0]), Column(FLOAT64, [1.0, 1.1])
    assert _hash([f32], [FLOAT32], [0], 0)[0] == _hash([f64], [FLOAT64], [0], 0)[0]
    assert _equal(FLOAT32, f32, 0, FLOAT64, f64, 0) == 1
    assert _equal(FLOAT32, f32, 0, FLOAT64, f64, 1) == 0
    x, y = Column(BYTES, [b"x"]), Column(BYTES, [b"x", b"y"])
    assert _hash([x], [BYTES], [0], 0)[0] == _hash([y], [BYTES], [0], 0)[0]
    assert _equal(BYTES, x, 0, BYTES, y, 0) == 1 and _equal(BYTES, x, 0, BYTES, y, 1) == 0


def test_hash_row_bytes_layout():
    # util/codec/codec.go:230-233,318-333: flag compactBytesFlag (2) then the raw cell bytes; FLOAT: floatFlag (5) + float64(f)
    s = Column(BYTES, [b"", b"abc", None, b"\x00\xff" * 40])
    for row, v in enumerate([b"", b"abc", None, b"\x00\xff" * 40]):
        h, hn = _hash([s], [BYTES], [0], row)
        assert (h, hn) == ((fnv1_64(bytes([0])), 1) if v is None else (fnv1_64(bytes([2]) + v), 0))
    f = Column(FLOAT32, np.array([0.1, -2.5], dtype=np.float32))
    for row in range(2):
        assert _hash([f], [FLOAT32], [0], row)[0] == fnv1_64(bytes([5]) + np.float64(f.values[row]).tobytes())
    # a string never equals an integer or a double with the same bits (flags differ: 2 vs 8 / 5)
    i = Column(INT64, [0x6162])
    assert _equal(BYTES, Column(BYTES, [b"ba"]), 0, INT64, i, 0) == 0


def py_join(btypes, bcols, ptypes, pcols, bkeys, pkeys):
    """independent restatement: key = tuple of (class, value) with FLOAT widened; inner join, (probe asc, build insertion asc)"""
    def kv(tp, col, r):
        if not col.not_null()[r]:
            return None
        if tp == BYTES:
            return ("s", col.values[r])
        if tp in (FLOAT32, FLOAT64):
            return ("f", np.float64(col.values[r]).tobytes())
        v = int(col.values[r])
        return ("u" if tp == UINT64 and v >= (1 << 63) else "i", v)
    table = defaultdict(list)
    for r in range(bcols[0].length):
        k = tuple(kv(btypes[c], bcols[c], r) for c in bkeys)
        if None not in k:
            table[k].append(r)
    out = []
    for r in range(pcols[0].length):
        k = tuple(kv(ptypes[c], pcols[c], r) for c in pkeys)
        if None in k:
            continue
        for br in table.get(k, ()):
            out.append((r, br))
    return out


def test_join_on_string_and_float_keys_matches_python_restatement():
    rng = np.random.default_rng(5)
    nb, npr = 400, 1500
    words = [b"", b"a", b"ab", b"abc", b"b" * 33, b"\x00", b"\x00\x00", b"xyz" * 100]
    bs = [words[i] if rng.random() > 0.1 else None for i in rng.integers(0, len(words), nb)]
    ps = [words[i] if rng.random() > 0.1 else None for i in rng.integers(0, len(words), npr)]
    bf = Column(FLOAT32, rng.integers(0, 4, nb).astype(np.float32) * 0.1, rng.random(nb) > 0.1)
    pf = Column(FLOAT64, rng.integers(0, 4, npr).astype(np.float32).astype(np.float64) * np.float64(np.float32(0.1)), rng.random(npr) > 0.1)
    # float32(k * 0.1f) widened == the float64 product only when the float32 product is exact; use the widened float32 values
    pf = Column(FLOAT64, (rng.integers(0, 4, npr).astype(np.float32) * np.float32(0.1)).astype(np.float64), rng.random(npr) > 0.1)
    bcols = [Column(BYTES, bs), bf, Column(INT64, np.arange(nb))]
    pcols = [pf, Column(BYTES, ps), Column(INT64, np.arange(npr))]
    bt, pt = [BYTES, FLOAT32, INT64], [FLOAT64, BYTES, INT64]
    for bk, pk in (([0], [1]), ([1], [0]), ([0, 1], [1, 0])):
        got = O.hash_join(0, False, bt, bcols, pt, pcols, bk, pk)
        want = py_join(bt, bcols, pt, pcols, bk, pk)
        assert got.num_rows() == len(want) and len(want) > 0
        assert [(int(p), int(b)) for p, b in zip(got.cols[2].values, got.cols[5].values)] == want


def test_agg_string_group_by_and_string_float_arguments():
    # executor/aggfuncs: maxMin4String / firstRow4String / countOriginal4String (func_max_min.go:312-376, func_first_row.go:193-238),
    # maxMin4Float32 / firstRow4Float32; GROUP BY a string column (HashGroupKey ETString, codec.go:735-743)
    g = Column(BYTES, [b"a", b"b", None, b"a", b"", b"b", None, b"a"])
    s = Column(BYTES, [b"pear", None, b"kiwi", b"apple", b"fig", b"zoo", b"", b"pea"])
    f = Column(FLOAT32, np.array([1.5, 2.5, 0.25, -1.0, 9.0, 2.25, 7.0, 3.0], dtype=np.float32), [True, True, True, True, False, True, True, True])
    funcs = [(FIRSTROW, 0), (COUNT, 1), (MAX, 1), (MIN, 1), (FIRSTROW, 1), (MAX, 2), (MIN, 2), (SUM, 2), (AVG, 2), (FIRSTROW, 2)]
    rc, out = O.hash_agg([BYTES, BYTES, FLOAT32], [g, s, f], [0], funcs)
    assert rc == 0
    rows = {r[0]: r[1:] for r in out.rows()}
    assert rows[b"a"] == (3, b"pear", b"apple", b"pear", 3.0, -1.0, 3.5, 3.5 / 3, 1.5)
    assert rows[b"b"] == (1, b"zoo", b"zoo", None, 2.5, 2.25, 4.75, 2.375, 2.5)
    assert rows[None] == (2, b"kiwi", b"", b"kiwi", 7.0, 0.25, 7.25, 3.625, 0.25)
    assert rows[b""] == (1, b"fig", b"fig", b"fig", None, None, None, None, None)
    assert [c.tp for c in out.cols] == [BYTES, INT64, BYTES, BYTES, BYTES, FLOAT32, FLOAT32, FLOAT64, FLOAT64, FLOAT32]
    # no GROUP BY, empty input: the default row (COUNT 0, NULLs), also for string / FLOAT result columns
    e = [Column(BYTES, []), Column(FLOAT32, np.zeros(0, dtype=np.float32))]
    rc, out = O.hash_agg([BYTES, FLOAT32], e, [], [(COUNT, 0), (MAX, 0), (MIN, 1)])
    assert rc == 0 and out.rows() == [(0, None, None)]


@pytest.mark.parametrize("workers", [1, 3])
def test_agg_string_partial_final_split_is_result_neutral(workers):
    rng = np.random.default_rng(11)
    n = 5000
    keys = [b"k%d" % v for v in rng.integers(0, 50, n)]
    vals = [(b"v%05d" % v) if rng.random() > 0.2 else None for v in rng.integers(0, 10000, n)]
    funcs = [(FIRSTROW, 0), (COUNT, 1), (MAX, 1), (MIN, 1)]
    rc, out = O.hash_agg([BYTES, BYTES], [Column(BYTES, keys), Column(BYTES, vals)], [0], funcs, n_partial_workers=workers)
    assert rc == 0
    want = defaultdict(list)
    for k, v in zip(keys, vals):
        want[k].append(v)
    got = {r[0]: r[1:] for r in out.rows()}
    assert set(got) == set(want)
    for k, vs in want.items():
        nn = [v for v in vs if v is not None]
        assert got[k] == (len(nn), max(nn) if nn else None, min(nn) if nn else None)
