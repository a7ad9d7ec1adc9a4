"""CPU suite: both ends of the nullable region exchange (csrc/partition.cu) under the emulation build of tests/emu — the mask
word and effective selection a pushing rank packs (k_pack_null_mask), and tq_region_gather, which copies the published
regions into contiguous columns and expands the mask word into NULL bitmaps.  Regions of 0, 1, 63, 64 and 65 rows put
region starts and ends on and off the 32-row bitmap words and 64-row groups; overflowed slots fail without a write."""
import ctypes as C
import itertools

import numpy as np
import pytest

import exchange_ref as X
import region_outer_ref as R
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)
from tinysql_b200 import _lib as L

COUNTS = [0, 1, 63, 64, 65]


class _DCol(C.Structure):
    """tq::DCol (csrc/common.cuh): a device column as the kernels see it"""
    _fields_ = [("data", C.c_void_p), ("bm", C.c_void_p)]


def _pack_null_mask(lib):
    """tq::pack_null_mask (csrc/scatter.cuh), which the product reaches only from the push in join.cu: the emulation library
    exports the internal C++ functions of the sources it compiles, so the test calls this one by its C++ symbol"""
    fn = getattr(lib, "_ZN2tq14pack_null_maskEPKNS_4DColEiiPKhlPmPhPv")
    fn.restype = C.c_int32
    fn.argtypes = [C.POINTER(_DCol), C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1000])
def test_emu_pack_null_mask(emu, n):
    """bit c of mask[r] = column c of row r is NOT NULL (columns without a bitmap: 1); sel_out = selected AND key NOT NULL,
    for the key in column 0 and in the last column"""
    rng = np.random.default_rng(n)
    cols = [rng.integers(0, 1 << 62, n).astype(np.uint64) for _ in range(3)]
    nns = [rng.random(n) >= 0.3, None, rng.random(n) >= 0.5]
    for key_col, with_sel in itertools.product((0, 2), (False, True)):
        sel = rng.random(n) >= 0.25 if with_sel else None
        src = R.Source(emu, cols, nns, sel)
        mask, sel_out = X.Buf(emu, n * 8 + 64), X.Buf(emu, n + 64)
        try:
            dcols = (_DCol * 3)(*[_DCol(src.ptrs[c], src.bms[c]) for c in range(3)])
            st = _pack_null_mask(emu)(dcols, 3, key_col, src.sel, n, mask.addr(), sel_out.addr(), None)
            assert st == L.TQ_OK
            want = sum((nn if nn is not None else np.ones(n, bool)).astype(np.uint64) << np.uint64(c) for c, nn in enumerate(nns))
            got = mask.get()
            assert np.array_equal(got[:n], want)
            assert np.all(got[n:] == X.SENTINEL), "a write past n mask words"
            want_sel = (sel if sel is not None else np.ones(n, bool)) & (nns[key_col] if nns[key_col] is not None else True)
            gs = sel_out.get(np.uint8)
            assert np.array_equal(gs[:n], want_sel.astype(np.uint8))
            assert np.all(gs[n:] == X.SENTINEL_BYTE)
        finally:
            src.free()
            mask.free()
            sel_out.free()


def _regions(lib, rng, counts, ncols, has_mask, cap):
    """one destination's W regions filled as the push leaves them: rows (+ mask words) and published slots"""
    W = len(counts)
    reg = X.Regions(lib, W, ncols + has_mask, cap)
    put = lambda a, g, c: reg.buf.put(a, reg.region_ptr(0, 0, g, c) - reg.buf.addr())
    rows, nns = [], []
    for g, m in enumerate(counts):
        v = [rng.integers(0, 1 << 62, m).astype(np.uint64) for _ in range(ncols)]
        nn = [rng.random(m) >= 0.4 for _ in range(ncols)]
        for c in range(ncols):
            put(v[c], g, c)
        if has_mask and m:
            put(sum(nn[c].astype(np.uint64) << np.uint64(c) for c in range(ncols)), g, ncols)
        rows.append(v)
        nns.append(nn if has_mask else [np.ones(m, bool)] * ncols)
    return reg, rows, nns


def _publish(reg, counts, epoch=1):
    slots = np.array([[c, epoch] for c in counts], np.uint64).reshape(-1)
    reg.buf.put(slots, reg.slot_ptr(0, 0, 0) - reg.buf.addr())


@pytest.mark.parametrize("has_mask", [0, 1])
@pytest.mark.parametrize("W", [1, 2, 3])
def test_emu_region_gather_counts(emu, W, has_mask):
    """every combination of region sizes from {0, 1, 63, 64, 65} (W <= 2; a sample at W = 3): the rows in region order,
    bitmaps with the mask's bits and 0 past the last row up to its 64-row group, nothing written past them"""
    rng = np.random.default_rng(10 * W + has_mask)
    combos = list(itertools.product(COUNTS, repeat=W))
    if W == 3:
        combos = [combos[i] for i in rng.choice(len(combos), 20, replace=False)] + [(65, 65, 65), (0, 0, 0)]
    ncols = 3 if has_mask else 2
    for counts in combos:
        reg, rows, nns = _regions(emu, rng, counts, ncols, has_mask, 65)
        _publish(reg, counts)
        out = R.GuardedCols(emu, ncols, 65 * W, True)
        try:
            st, n = R.gather(emu, W, reg.slot_ptr(0, 0, 0), 65, ncols, has_mask, reg.region_table(0, 0), out)
            assert st == L.TQ_OK and n == sum(counts), (counts, st, n)
            assert all(out.arr[c].length == n for c in range(ncols))
            assert out.guards_ok(n), f"{counts}: a write past the rows / bitmap words"
            for c, (v, nn) in enumerate(out.read(n)):
                assert np.array_equal(v, np.concatenate([r[c] for r in rows])), f"{counts}: column {c} values"
                want = np.concatenate([x[c] for x in nns] + [np.zeros((-n) % 64, bool)])
                assert np.array_equal(nn, want), f"{counts}: column {c} bitmap (bits past the last row must be 0)"
        finally:
            out.free()
            reg.free()


def test_emu_region_gather_without_bitmaps_and_empty(emu):
    """NULL output bitmaps: only values are written; no rows at all: n = 0, nothing written"""
    rng = np.random.default_rng(3)
    reg, rows, _ = _regions(emu, rng, [5, 0, 70], 2, 1, 70)
    _publish(reg, [5, 0, 70])
    out = R.GuardedCols(emu, 2, 200, False)
    try:
        st, n = R.gather(emu, 3, reg.slot_ptr(0, 0, 0), 70, 2, 1, reg.region_table(0, 0), out)
        assert st == L.TQ_OK and n == 75
        assert out.guards_ok(75)
        for c, (v, nn) in enumerate(out.read(75)):
            assert nn is None and np.array_equal(v, np.concatenate([r[c] for r in rows]))
        _publish(reg, [0, 0, 0])
        out2 = R.GuardedCols(emu, 2, 64, True)
        st, n = R.gather(emu, 3, reg.slot_ptr(0, 0, 0), 70, 2, 1, reg.region_table(0, 0), out2)
        assert st == L.TQ_OK and n == 0 and out2.untouched()
        out2.free()
    finally:
        out.free()
        reg.free()


@pytest.mark.parametrize("bad", ["overflowed", "over_cap", "out_cap"])
def test_emu_region_gather_refusals(emu, bad):
    """a slot reading ~0 (an overflowed push) or more than region_cap: TQ_ERR_OOM; more rows than out_cap:
    TQ_ERR_INVALID_ARG; bad shapes: TQ_ERR_INVALID_ARG.  Nothing is written to the outputs."""
    rng = np.random.default_rng(4)
    counts = [64, 65, 1]
    reg, _, _ = _regions(emu, rng, counts, 2, 1, 65)
    published = {"overflowed": [64, (1 << 64) - 1, 1], "over_cap": [64, 66, 1], "out_cap": counts}[bad]
    _publish(reg, published)
    out = R.GuardedCols(emu, 2, 200, True)
    try:
        st, n = R.gather(emu, 3, reg.slot_ptr(0, 0, 0), 65, 2, 1, reg.region_table(0, 0), out, out_cap=129 if bad == "out_cap" else None)
        assert st == (L.TQ_ERR_INVALID_ARG if bad == "out_cap" else L.TQ_ERR_OOM), st
        assert n == -1 and out.untouched(), "a refused gather wrote"
        for args in ((0, 65, 2, 1), (9, 65, 2, 1), (3, 0, 2, 1), (3, 65, 4, 1), (3, 65, 0, 0), (3, 65, 2, 2)):
            st, _ = R.gather(emu, args[0], reg.slot_ptr(0, 0, 0), args[1], args[2], args[3], reg.region_table(0, 0), out)
            assert st == L.TQ_ERR_INVALID_ARG, args
        assert out.untouched()
    finally:
        out.free()
        reg.free()
