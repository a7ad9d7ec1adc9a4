"""CPU suite: the broadcast push's copy (csrc/partition.cu: broadcast_rows / k_broadcast) under the emulation build of
tests/emu, against numpy.  Every destination gets, in dist.BroadcastJoin's layout (a sentinel guard after every area):
8-byte values, bitmap words (copied, or all ones for a column without a bitmap on a nullable side), BYTES offsets rebased to
0 and the cells behind them — empty cells, NULL cells, and a sliced source whose offsets[0] != 0 at every byte alignment.
Row counts 0, 1, 63, 64, 65 and 4097 put the ends on and off the 64-row bitmap words and the 16-byte stores; a byte area
exactly full is copied, one byte short sets the overflow flag and receives nothing."""
import ctypes as C

import numpy as np
import pytest

import exchange_ref as X
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)
from tinysql_b200 import _lib as L
from tinysql_b200.dist import BroadcastJoin, RegionLayout

GUARD = 64
COUNTS = [0, 1, 63, 64, 65, 4097]
I64, U64, F64, BYTES = L.TQ_TYPE_INT64, L.TQ_TYPE_UINT64, L.TQ_TYPE_FLOAT64, L.TQ_TYPE_BYTES


def _broadcast_rows(lib):
    """tq::broadcast_rows (csrc/scatter.cuh), called by its C++ symbol: the emulation library exports the internal functions"""
    fn = getattr(lib, "_ZN2tq14broadcast_rowsEiPK9tq_columnPKiiliPKPvPKlPjPyS5_")
    fn.restype = C.c_int32
    fn.argtypes = [C.c_int, C.POINTER(L.TQColumn), C.POINTER(C.c_int32), C.c_int, C.c_int64, C.c_int, C.c_void_p, C.POINTER(C.c_int64),
                   C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


def _cells(rng, n, null_frac=0.2):
    """n byte strings of 0..40 bytes (some empty) and their NOT-NULL flags (a NULL cell is empty)"""
    nn = rng.random(n) >= null_frac
    cells = [bytes(rng.integers(0, 256, rng.integers(0, 41), dtype=np.uint8)) if ok and rng.random() > 0.15 else b"" for ok in nn]
    return cells, nn


class _Side:
    """one source's columns in emulated device memory; a BYTES column's cells sit `lead` bytes into its allocation, so
    offsets[0] == lead"""

    def __init__(self, lib, types, vals, nns, lead):
        self.bufs, self.arr = [], (L.TQColumn * len(types))()
        n = len(vals[0])
        for c, (t, v, nn) in enumerate(zip(types, vals, nns)):
            self.arr[c].length = n
            if t == BYTES:
                offs = lead + np.concatenate([[0], np.cumsum([len(x) for x in v])]).astype(np.int64)
                raw = np.frombuffer(b"\xee" * lead + b"".join(v), np.uint8)
                self.arr[c].offsets = self._put(lib, offs)
                self.arr[c].data = self._put(lib, raw) if raw.size else None
            else:
                self.arr[c].data = self._put(lib, np.asarray(v, np.uint64))
            if nn is not None:
                self.arr[c].null_bitmap = self._put(lib, X.bitmap_words(nn))

    def _put(self, lib, a):
        b = X.Buf(lib, max(a.nbytes, 8), None)
        b.put(a)
        self.bufs.append(b)
        return b.addr()

    def free(self):
        for b in self.bufs:
            b.free()


def _run(lib, types, vals, nns, nullable, n_parts, byte_caps, lead=0, guard=GUARD):
    """broadcast_rows of one source into n_parts emulated destinations: (status, rows[q], overflow, layout, buffer).  An odd
    guard puts every other area off 16-byte alignment, where the copy stores word by word"""
    n = len(vals[0])
    table = BroadcastJoin.table_of(types, max(n, 1), byte_caps, nullable)
    lay = RegionLayout(lib, L, n_parts, [table], pad_rows=guard)
    buf = X.Buf(lib, n_parts * lay.bytes)
    lay.bases = [buf.addr(d * lay.bytes) for d in range(n_parts)]
    side = _Side(lib, types, vals, nns, lead)
    rows, ovf = X.Buf(lib, 64), X.Buf(lib, 8, 0)
    try:
        dest, _ = lay.push_tables(0, 0)
        caps = (C.c_int64 * len(types))(*[int(b or 0) for b in byte_caps])
        st = _broadcast_rows(lib)(len(types), side.arr, (C.c_int32 * len(types))(*types), int(nullable), n, n_parts, dest, caps, rows.addr(),
                                  ovf.addr(), None)
        return st, rows.get(np.uint32)[:n_parts], int(ovf.get()[0]), lay, buf
    finally:
        side.free()
        rows.free()
        ovf.free()


def _area(lay, buf, dst, a, dtype=np.uint64):
    """area a of source 0 on destination dst, its guard words included"""
    start = lay.region_ptr(dst, 0, 0, a) - buf.addr()
    end = (lay.region_ptr(dst, 0, 0, a + 1) if a + 1 < lay.ncols[0] else lay.region_ptr(dst, 0, 0, 0) + lay.stride[0] * 8) - buf.addr()
    return buf.get(dtype, start, end - start)


def _check(lay, buf, dst, types, vals, nns, nullable, n, byte_caps, overflowed=()):
    """every area of destination dst against numpy, and the sentinel everywhere past what the rows fill"""
    a = 0
    for c, t in enumerate(types):
        if t == BYTES:
            off = _area(lay, buf, dst, a).view(np.int64)
            want = np.concatenate([[0], np.cumsum([len(x) for x in vals[c]])]).astype(np.int64)
            assert np.array_equal(off[:n + 1], want), (c, "offsets")
            assert np.all(off[n + 1:].view(np.uint64) == X.SENTINEL), (c, "past the offsets")
            cells = _area(lay, buf, dst, a + 1, np.uint8)
            raw = np.frombuffer(b"".join(vals[c]), np.uint8)
            if c in overflowed:
                assert np.all(cells == X.SENTINEL_BYTE), (c, "an overflowed column's cells were written")
            else:
                assert np.array_equal(cells[:raw.size], raw), (c, "cells")
                assert np.all(cells[raw.size:] == X.SENTINEL_BYTE), (c, "past the cells")
            a += 2
        else:
            v = _area(lay, buf, dst, a)
            assert np.array_equal(v[:n], np.asarray(vals[c], np.uint64)), (c, "values")
            assert np.all(v[n:] == X.SENTINEL), (c, "past the values")
            a += 1
        if nullable:
            bm = _area(lay, buf, dst, a, np.uint8)
            nw = (n + 63) // 64
            got = np.unpackbits(bm[:nw * 8], bitorder="little").astype(bool)[:n]
            want = np.ones(n, bool) if nns[c] is None else np.asarray(nns[c], bool)
            assert np.array_equal(got, want), (c, "bitmap")
            assert np.all(bm[nw * 8:] == X.SENTINEL_BYTE), (c, "past the bitmap words")
            a += 1


def _side(rng, n):
    """INT64 with NULLs, BYTES with NULLs and empty cells, UINT64 (sign bit set) without a bitmap, FLOAT64"""
    types = [I64, BYTES, U64, F64]
    cells, cnn = _cells(rng, n)
    vals = [rng.integers(-(1 << 62), 1 << 62, n).astype(np.int64).view(np.uint64), cells,
            rng.integers(0, 1 << 63, n, dtype=np.uint64) | np.uint64(1 << 63), rng.random(n).view(np.uint64)]
    nns = [rng.random(n) >= 0.3, cnn, None, rng.random(n) >= 0.1]
    return types, vals, nns


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("nullable", [False, True])
def test_emu_broadcast_copy(emu, n, nullable):
    """1, 2 and 3 destinations, sliced sources at leads 0, 3 and 13, areas on and off 16-byte alignment: every area exact,
    nothing past it"""
    rng = np.random.default_rng(n + 7 * nullable)
    types, vals, nns = _side(rng, n)
    if not nullable:
        nns = [None] * len(types)
    nbytes = sum(len(x) for x in vals[1])
    for n_parts, lead, guard in ((1, 0, GUARD), (2, 3, GUARD - 1), (3, 13, GUARD)):
        caps = [None, nbytes + 17, None, None]
        st, rows, ovf, lay, buf = _run(emu, types, vals, nns, nullable, n_parts, caps, lead, guard)
        try:
            assert st == L.TQ_OK
            assert list(rows) == [n] * n_parts and ovf == 0
            for d in range(n_parts):
                _check(lay, buf, d, types, vals, nns, nullable, n, caps)
        finally:
            buf.free()


@pytest.mark.parametrize("n", [1, 64, 4097])
def test_emu_broadcast_byte_area_edges(emu, n):
    """two BYTES columns: the first fills its byte area exactly (copied), the second is one byte short (overflow = 1, its
    cells not written, the other column's still are)"""
    rng = np.random.default_rng(100 + n)
    a, _ = _cells(rng, n, 0.0)
    b, _ = _cells(rng, n, 0.0)
    if not any(b):
        b[0] = b"x"
    types, vals, nns = [BYTES, I64, BYTES], [a, np.arange(n, dtype=np.uint64), b], [None, None, None]
    na, nb = sum(map(len, a)), sum(map(len, b))
    for caps, over in (([na, None, nb], ()), ([na, None, nb - 1], (2,))):
        st, rows, ovf, lay, buf = _run(emu, types, vals, nns, False, 2, caps, lead=5)
        try:
            assert st == L.TQ_OK and list(rows) == [n, n]
            assert ovf == (1 if over else 0)
            for d in range(2):
                _check(lay, buf, d, types, vals, nns, False, n, caps, over)
        finally:
            buf.free()
