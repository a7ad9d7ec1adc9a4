"""CPU suite: the multi-GPU ORDER BY's device pieces under the emulation build of tests/emu.

- k_range_dest (tq::range_dest) against the routing twin of tests/region_sort_ref.py — sort_ref.key_words per ByItem, most
  significant first, then the tie word — over NULLs with ASC and DESC, -0.0 next to +0.0, the INT64 limits, UINT64 >= 2^63,
  strings that share 8-, 16- and 17-byte prefixes, end in zero bytes or are "" next to NULL, and 1..8 ByItems; every row
  equal (each destination gets exactly the rows whose tie words fall between its splitters); shards of 0..65 rows; and the
  destination never decreases along the routing order.
- The sample gather (tq::sample_rows): positions, values, NOT-NULL bits, string cells and tie words against the twin.
- tq_sort_put_regions against sort_ref.sort_rows of the regions concatenated in source order, and its refusals."""
import ctypes as C

import numpy as np
import pytest

import exchange_ref as X
import region_sort_ref as RS
import sort_ref as SR
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)
from test_emu_region_agg import _Dev
from tinysql_b200 import _lib as L

I64, U64, F64, F32, BYTES = L.TQ_TYPE_INT64, L.TQ_TYPE_UINT64, L.TQ_TYPE_FLOAT64, L.TQ_TYPE_FLOAT32, L.TQ_TYPE_BYTES
COUNTS = [0, 1, 63, 64, 65]
M64 = (1 << 64) - 1
PUSH_FAILED = 0xFFFFFFFF00000000


class _RangeBy(C.Structure):
    """tq::RangeBy (csrc/scatter.cuh)"""
    _fields_ = [("type", C.c_int), ("desc", C.c_int), ("data", C.c_void_p), ("off", C.c_void_p), ("bytes", C.c_void_p), ("bm", C.c_void_p)]


class _SampleOut(C.Structure):
    """tq::SampleOut (csrc/scatter.cuh)"""
    _fields_ = [("data", C.c_void_p * 8), ("off", C.c_void_p * 8), ("bytes", C.c_void_p * 8), ("bm", C.c_void_p * 8),
                ("byte_cap", C.c_uint64 * 8), ("tie", C.c_void_p)]


def _range_dest(lib):
    fn = getattr(lib, "_ZN2tq10range_destEPKNS_7RangeByES2_iPKmPKliilPhPv")
    fn.restype = C.c_int32
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_void_p]
    return fn


def _sample_rows(lib):
    fn = getattr(lib, "_ZN2tq11sample_rowsEPKNS_7RangeByEillmiRKNS_9SampleOutEPv")
    fn.restype = C.c_int32
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_uint64, C.c_int, C.POINTER(_SampleOut), C.c_void_p]
    return fn


def _by(dev, tp, vals, desc, lead=5):
    """a ByItem column of Python values (None = NULL) in emulated device memory; a BYTES column's offsets start at `lead`"""
    nn = [v is not None for v in vals]
    b = _RangeBy(tp, int(desc), None, None, None, dev.bitmap(nn) if vals else None)
    if tp == BYTES:
        cells = [v or b"" for v in vals]
        off = lead + np.concatenate([[0], np.cumsum([len(x) for x in cells])]).astype(np.int64)
        b.off = dev.put(off).addr()
        b.bytes = dev.put(np.frombuffer(b"\xee" * lead + b"".join(cells) + b"\0" * 8, np.uint8)).addr()
    else:
        dt = {I64: np.int64, U64: np.uint64, F64: np.float64}[tp]
        b.data = dev.put(np.array([0 if v is None else v for v in vals], dt).view(np.uint64) if vals else np.zeros(1, np.uint64)).addr()
    return b


def _route(lib, by, rows, spl, spl_ties, pos, src_rank):
    """dest[] from tq::range_dest and from the twin; rows / spl: per ByItem the Python values"""
    n = len(rows[0]) if rows else 0
    want = RS.range_dest(by, rows, [RS.tie(src_rank, i) for i in range(n)], [[s[p] for p in pos] for s in spl], [spl_ties[p] for p in pos])
    if n == 0:                                     # the push sends no rows and launches nothing
        return [], want
    dev = _Dev(lib)
    try:
        rb = (_RangeBy * max(len(by), 1))(*[_by(dev, t, v, d) for (t, d), v in zip(by, rows)])
        sb = (_RangeBy * max(len(by), 1))(*[_by(dev, t, v, d, lead=3) for (t, d), v in zip(by, spl)])
        tie = dev.put(np.array(spl_ties, np.uint64)).addr() if pos else None
        hp = (C.c_int64 * max(len(pos), 1))(*pos)
        out = X.Buf(lib, n + 64)
        dev.bufs.append(out)
        st = _range_dest(lib)(C.addressof(rb), C.addressof(sb), len(by), tie, C.addressof(hp) if pos else None, len(pos), src_rank, n, out.addr(), None)
        assert st == L.TQ_OK
        got = out.get(np.uint8)
        assert np.all(got[n:] == X.SENTINEL_BYTE), "a write past the rows"
        return got[:n].tolist(), want
    finally:
        dev.free()


def _splitters(rng, by, pool, n_parts, k=24):
    """a sorted sample (per ByItem values, tie words) drawn from the value pools, and n_parts - 1 non-decreasing positions"""
    vals = [[p[i] for i in rng.integers(0, len(p), k)] for p in pool]
    ties = [RS.tie(int(r), int(i)) for r, i in zip(rng.integers(0, 4, k), rng.integers(0, 70, k))]
    keys = RS.routing_keys(by, vals, ties)
    order = sorted(range(k), key=lambda i: keys[i])
    vals = [[v[i] for i in order] for v in vals]
    ties = [ties[i] for i in order]
    pos = sorted(int(x) for x in rng.integers(0, k, n_parts - 1))
    return vals, ties, pos


def _pools():
    """the edge values per type"""
    s = [None, b"", b"\0", b"a", b"a\0", b"abcdefgh", b"abcdefgh\0", b"abcdefghij", b"abcdefghijklmnop", b"abcdefghijklmnopq",
         b"abcdefghijklmnoq", b"abcdefghijklmnop\0", b"b", b"\xff" * 20]
    return {
        I64: [None, SR.INT64_MIN, SR.INT64_MIN + 1, -1, 0, 1, SR.INT64_MAX],
        U64: [None, 0, 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, SR.UINT64_MAX],
        F64: [None, -0.0, 0.0, -1.5, 1.5, float("-inf"), float("inf"), SR.DBL_TRUE_MIN, -SR.DBL_MAX],
        BYTES: s,
    }


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("tp", [I64, U64, F64, BYTES])
def test_emu_range_dest_one_item(emu, tp, n):
    """one ByItem of every type, ASC and DESC, 1..8 destinations: k_range_dest == the twin"""
    rng = np.random.default_rng(tp * 100 + n)
    pool = _pools()[tp]
    for desc in (False, True):
        by = [(tp, desc)]
        for n_parts in (1, 2, 3, 8):
            rows = [[pool[i] for i in rng.integers(0, len(pool), n)]]
            spl, ties, pos = _splitters(rng, by, [pool], n_parts)
            got, want = _route(emu, by, rows, spl, ties, pos, src_rank=int(rng.integers(0, 4)))
            assert got == want, (tp, desc, n_parts)


@pytest.mark.parametrize("n_by", range(1, 9))
def test_emu_range_dest_many_items(emu, n_by):
    """1..8 ByItems of mixed types and directions over few distinct values, so later items and the tie word decide"""
    rng = np.random.default_rng(n_by)
    pools = _pools()
    types = [[I64, U64, F64, BYTES][i % 4] for i in range(n_by)]
    by = [(t, bool(rng.integers(0, 2))) for t in types]
    pool = [pools[t][:4] for t in types]
    for n in (65, 200):
        rows = [[p[i] for i in rng.integers(0, len(p), n)] for p in pool]
        for n_parts in (2, 5, 8):
            spl, ties, pos = _splitters(rng, by, pool, n_parts)
            got, want = _route(emu, by, rows, spl, ties, pos, src_rank=1)
            assert got == want


@pytest.mark.parametrize("n", [63, 64, 65, 400])
def test_emu_range_dest_all_equal_splits_by_tie(emu, n):
    """every key equal: the splitters are (key, tie) points inside the run, so destination d gets exactly the rows whose tie
    words fall between its splitters — no destination receives everything"""
    by = [(I64, False), (BYTES, True)]
    rows = [[7] * n, [b"same"] * n]
    src = 2
    cuts = [n // 4, n // 2, 3 * n // 4]
    spl = [[7] * 3, [b"same"] * 3]
    ties = [RS.tie(src, c) for c in cuts]
    got, want = _route(emu, by, rows, spl, ties, [0, 1, 2], src_rank=src)
    assert got == want
    assert got == [sum(1 for c in cuts if c <= i) for i in range(n)]
    assert max(np.bincount(got)) < n


def test_emu_range_dest_no_splitters(emu):
    """no splitter rows (n_split = 0): every row to destination 0"""
    got, _ = _route(emu, [(I64, False)], [[3, None, -1]], [[]], [], [], src_rank=0)
    assert got == [0, 0, 0]


def test_emu_range_dest_monotone(emu):
    """property: along the routing order (the rows sorted by the twin's keys), the destination never decreases"""
    rng = np.random.default_rng(9)
    pools = _pools()
    by = [(F64, True), (BYTES, False), (U64, False)]
    pool = [pools[F64], pools[BYTES], pools[U64][:3]]
    n = 300
    rows = [[p[i] for i in rng.integers(0, len(p), n)] for p in pool]
    for n_parts in (2, 4, 8):
        spl, ties, pos = _splitters(rng, by, pool, n_parts, k=40)
        got, want = _route(emu, by, rows, spl, ties, pos, src_rank=3)
        assert got == want
        keys = RS.routing_keys(by, rows, [RS.tie(3, i) for i in range(n)])
        order = sorted(range(n), key=lambda i: keys[i])
        d = [got[i] for i in order]
        assert all(a <= b for a, b in zip(d, d[1:]))


@pytest.mark.parametrize("n,n_samples", [(1, 16), (63, 16), (64, 64), (65, 1000), (1000, 37)])
def test_emu_sample_gather(emu, n, n_samples):
    """m = min(n, n_samples) distinct rows at the twin's positions: values, NOT-NULL bits, cells and tie words"""
    rng = np.random.default_rng(n)
    pools = _pools()
    types = [I64, BYTES, F64]
    vals = [[pools[t][i] for i in rng.integers(0, len(pools[t]), n)] for t in types]
    m, seed, src = min(n, n_samples), 0x1234, 5
    dev = _Dev(emu)
    try:
        by = (_RangeBy * 3)(*[_by(dev, t, v, False) for t, v in zip(types, vals)])
        out = _SampleOut()
        bufs = {}
        for b, t in enumerate(types):
            if t == BYTES:
                bufs[(b, "off")] = X.Buf(emu, (m + 1) * 8)
                bufs[(b, "bytes")] = X.Buf(emu, 4096)
                out.off[b], out.bytes[b], out.byte_cap[b] = bufs[(b, "off")].addr(), bufs[(b, "bytes")].addr(), 4096
            else:
                bufs[(b, "data")] = X.Buf(emu, m * 8)
                out.data[b] = bufs[(b, "data")].addr()
            bufs[(b, "bm")] = X.Buf(emu, (m + 255) // 256 * 32)
            out.bm[b] = bufs[(b, "bm")].addr()
        bufs["tie"] = X.Buf(emu, m * 8)
        out.tie = bufs["tie"].addr()
        dev.bufs += list(bufs.values())
        assert _sample_rows(emu)(C.addressof(by), 3, n, m, seed, src, C.byref(out), None) == L.TQ_OK
        pos = [RS.sample_pos(seed, src, j, n, m) for j in range(m)]
        assert len(set(pos)) == m and all(0 <= p < n for p in pos)
        assert bufs["tie"].get().tolist() == [RS.tie(src, p) for p in pos]
        for b, t in enumerate(types):
            want = [vals[b][p] for p in pos]
            nn = np.unpackbits(bufs[(b, "bm")].get(np.uint8), bitorder="little")[:m].astype(bool)
            assert nn.tolist() == [v is not None for v in want]
            if t == BYTES:
                off = bufs[(b, "off")].get(np.int64)[:m + 1]
                cells = bufs[(b, "bytes")].get(np.uint8)
                got = [cells[off[j]:off[j + 1]].tobytes() for j in range(m)]
                assert off[0] == 0 and got == [v or b"" for v in want]
            else:
                dt = {I64: np.int64, F64: np.float64}[t]
                got = bufs[(b, "data")].get(dt)[:m]
                assert [g for g, ok in zip(got.tolist(), nn) if ok] == [v for v in want if v is not None]
    finally:
        dev.free()


# ------------------------------------------------------------------------------------------------ tq_sort_put_regions
def _sort_handle(lib, types, by, offset=0, count=-1):
    tt = (C.c_int32 * len(types))(*types)
    bc = (C.c_int32 * max(len(by), 1))(*[c for c, _ in by])
    bd = (C.c_int32 * max(len(by), 1))(*[int(d) for _, d in by])
    d = L.TQSortDesc(len(types), tt, len(by), bc, bd, offset, count)
    h = C.c_void_p()
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    return h


def _regions(dev, types, sources, cap, epoch=1, slot_rows=None):
    """the regions of W sources in the range push's wire format (per column its words or offsets from 0, the mask word, the
    byte areas): (slots address, regions tq_column array)"""
    nc = len(types)
    regs = (L.TQColumn * (len(sources) * (nc + 1)))()
    slots = []
    for g, rows in enumerate(sources):
        k = len(rows)
        slots += [k if slot_rows is None else slot_rows[g], epoch]
        mask = np.zeros(max(k, 1), np.uint64)
        for c, t in enumerate(types):
            vals = [r[c] for r in rows]
            mask[:k] |= np.array([v is not None for v in vals], np.uint64) << np.uint64(c)
            e = regs[g * (nc + 1) + c]
            e.length = cap
            if t == BYTES:
                cells = [v or b"" for v in vals]
                off = np.zeros(cap + 1, np.int64)
                off[1:k + 1] = np.cumsum([len(x) for x in cells]) if k else []
                e.offsets = dev.put(off).addr()
                e.data = dev.put(np.frombuffer(b"".join(cells) + b"\0" * 8, np.uint8)).addr()
            else:
                dt = {I64: np.int64, U64: np.uint64, F64: np.float64}[t]
                a = np.zeros(cap, np.uint64)
                a[:k] = np.array([0 if v is None else v for v in vals], dt).view(np.uint64)
                e.data = dev.put(a).addr()
        regs[g * (nc + 1) + nc].length = cap
        regs[g * (nc + 1) + nc].data = dev.put(mask).addr()
    return dev.put(np.array(slots, np.uint64)).addr(), regs


def _drain(lib, h, types):
    """the handle's result via tq_sort_next (host copy): rows of Python values"""
    from tinysql_b200.chunk import Column, VarColumn
    cols = [VarColumn.empty(t, 4096, 1 << 16) if t == BYTES else Column.empty(t, 4096) for t in types]
    arr = (L.TQColumn * len(types))(*[c.tq() for c in cols])
    rows, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_sort_next(h, 4096, arr, C.byref(rows), C.byref(eof)))
    k = rows.value
    out = [c.head(k) if t == BYTES else Column(t, c.values[:k], c.not_null()[:k]) for c, t in zip(cols, types)]
    return RS.rows_of(out) if k else []


def _src_rows(rng, types, k):
    pools = _pools()
    return [tuple(pools[t][i] for t, i in zip(types, [rng.integers(0, len(pools[t])) for t in types])) for _ in range(k)]


@pytest.mark.parametrize("counts", [(0,), (1, 0, 65), (63, 64), (5, 0, 0, 9, 2, 0, 1, 40)])
def test_emu_sort_put_regions(emu, counts):
    """W regions put in source order, then sorted: == sort_ref.sort_rows of their concatenation, for ASC / DESC mixes, TopN
    windows and the empty case"""
    rng = np.random.default_rng(sum(counts) + len(counts))
    types = [BYTES, I64, F64, U64]
    sources = [_src_rows(rng, types, k) for k in counts]
    allrows = [r for s in sources for r in s]
    cap = max(max(counts), 1)
    for by, off, cnt in (([(0, False), (1, True)], 0, -1), ([(2, True), (3, False), (0, True)], 0, -1), ([(1, False)], 3, 17), ([], 0, 5)):
        dev = _Dev(emu)
        h = _sort_handle(emu, types, by, off, cnt)
        try:
            slots, regs = _regions(dev, types, sources, cap)
            L.check(emu.tq_sort_put_regions(h, len(sources), C.c_void_p(slots), cap, regs))
            L.check(emu.tq_sort_eof(h))
            got = _drain(emu, h, types)
            assert SR.canon_rows(got) == SR.canon_rows(SR.sort_rows(allrows, by, off, cnt)), by
        finally:
            emu.tq_sort_destroy(h)
            dev.free()


def test_emu_sort_put_regions_refusals(emu):
    """an overflowed source (~0) is TQ_ERR_OOM, a failed source returns its status, a FLOAT32 column is
    TQ_ERR_UNSUPPORTED_TYPE, a region without its area TQ_ERR_INVALID_ARG: each puts nothing"""
    rng = np.random.default_rng(1)
    types = [I64, BYTES]
    sources = [_src_rows(rng, types, 10), _src_rows(rng, types, 7)]
    for slot_rows, status in (([10, M64], L.TQ_ERR_OOM), ([PUSH_FAILED | L.TQ_ERR_OOM, 7], L.TQ_ERR_OOM),
                              ([10, PUSH_FAILED | L.TQ_ERR_INVALID_ARG], L.TQ_ERR_INVALID_ARG), ([11, 7], L.TQ_ERR_OOM)):
        dev = _Dev(emu)
        h = _sort_handle(emu, types, [(0, False)])
        try:
            slots, regs = _regions(dev, types, sources, 10, slot_rows=slot_rows)
            assert emu.tq_sort_put_regions(h, 2, C.c_void_p(slots), 10, regs) == status
            L.check(emu.tq_sort_eof(h))
            assert _drain(emu, h, types) == []
        finally:
            emu.tq_sort_destroy(h)
            dev.free()
    dev = _Dev(emu)
    try:
        slots, regs = _regions(dev, types, sources, 10)
        h = _sort_handle(emu, [F32, BYTES], [(0, False)])
        assert emu.tq_sort_put_regions(h, 2, C.c_void_p(slots), 10, regs) == L.TQ_ERR_UNSUPPORTED_TYPE
        emu.tq_sort_destroy(h)
        h = _sort_handle(emu, types, [(0, False)])
        regs[1].offsets = None
        assert emu.tq_sort_put_regions(h, 2, C.c_void_p(slots), 10, regs) == L.TQ_ERR_INVALID_ARG
        emu.tq_sort_destroy(h)
    finally:
        dev.free()
