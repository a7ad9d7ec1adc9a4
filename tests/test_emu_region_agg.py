"""CPU suite: the GROUP BY push's kernels (csrc/partition.cu) under the emulation build of tests/emu — the destination of a
partial row (k_group_dest) against its Python twin (tests/region_agg_ref.py), and the wide scatter into per-destination
regions with the mask word packed on the way (k_part_hist / k_part_scatter with the region policy, k_region_rows).  Regions
of 0, 1, 63, 64 and 65 rows put region ends on and off the 32-row bitmap words and 64-row groups; a cap one row short
overflows without a write past the cap."""
import ctypes as C
import itertools

import numpy as np
import pytest

import exchange_ref as X
import region_agg_ref as RA
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)
from tinysql_b200 import _lib as L
from tinysql_b200.dist import dest_rank_np

COUNTS = [0, 1, 63, 64, 65]


class _DCol(C.Structure):
    """tq::DCol (csrc/common.cuh)"""
    _fields_ = [("data", C.c_void_p), ("bm", C.c_void_p)]


def _group_dest(lib):
    """tq::group_dest (csrc/scatter.cuh), called by its C++ symbol: the emulation library exports the internal functions"""
    fn = getattr(lib, "_ZN2tq10group_destEPKNS_4DColEijliPhPv")
    fn.restype = C.c_int32
    fn.argtypes = [C.POINTER(_DCol), C.c_int, C.c_uint32, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
    return fn


def _scatter_to_regions(lib):
    """tq::scatter_to_regions (csrc/scatter.cuh); its RegionScratch is three DevBufs {void *p; size_t cap}"""
    fn = getattr(lib, "_ZN2tq18scatter_to_regionsEPKNS_4DColEiPKhliPKPmlPjPyRNS_13RegionScratchEPv")
    fn.restype = C.c_int32
    fn.argtypes = [C.POINTER(_DCol), C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


class _Dev:
    """host arrays in emulated device memory (sentinel-guarded by X.Buf)"""

    def __init__(self, lib):
        self.lib, self.bufs = lib, []

    def put(self, a, extra=64):
        a = np.ascontiguousarray(a)
        b = X.Buf(self.lib, a.nbytes + extra)
        b.put(a)
        self.bufs.append(b)
        return b

    def bitmap(self, nn):
        return None if nn is None else self.put(X.bitmap_words(nn)).addr()

    def free(self):
        for b in self.bufs:
            b.free()


def _items(rng, n, kinds):
    """GROUP BY columns of n rows: kind 'i' INT64, 'u' UINT64 (sign bit set half the time), 'r' REAL with both zeros; NULLs
    in every other item"""
    vals, nns, reals = [], [], []
    for g, k in enumerate(kinds):
        if k == "r":
            v = rng.choice(np.array([0.0, -0.0, 1.5, -2.25, np.inf], np.float64), n).view(np.uint64)
        elif k == "u":
            v = rng.integers(0, 1 << 63, n, dtype=np.uint64) | (rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63))
        else:
            v = rng.integers(-5, 5, n).astype(np.int64).view(np.uint64)
        vals.append(v)
        nns.append(rng.random(n) >= 0.3 if g % 2 == 0 else None)
        reals.append(k == "r")
    return vals, nns, reals


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1000])
def test_emu_group_dest_matches_twin(emu, n):
    """every item layout of 0..3 items over INT64 / UINT64 / REAL with NULLs, 1..8 destinations: k_group_dest == the twin;
    -0.0 and +0.0 rows share a destination; one NOT NULL item gives dest_rank_np; no item gives 0"""
    rng = np.random.default_rng(n)
    fn = _group_dest(emu)
    layouts = [()] + [tuple(p) for k in (1, 2, 3) for p in itertools.product("iur", repeat=k)]
    for kinds in layouts:
        vals, nns, reals = _items(rng, n, kinds)
        dev = _Dev(emu)
        try:
            items = (_DCol * max(len(kinds), 1))(*[_DCol(dev.put(v).addr(), dev.bitmap(nn)) for v, nn in zip(vals, nns)])
            real_mask = sum(1 << g for g, r in enumerate(reals) if r)
            for n_parts in (1, 2, 3, 8):
                out = X.Buf(emu, n + 64)
                try:
                    assert fn(items, len(kinds), real_mask, n, n_parts, out.addr(), None) == L.TQ_OK
                    got = out.get(np.uint8)
                    want = RA.group_dest(n, vals, nns, reals, n_parts)
                    assert np.array_equal(got[:n], want.astype(np.uint8)), (kinds, n_parts)
                    assert np.all(got[n:] == X.SENTINEL_BYTE)
                finally:
                    out.free()
        finally:
            dev.free()
    # the join's rank for one NOT NULL key, and +0.0 / -0.0 as one item (alone and second of two)
    k = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64)
    assert np.array_equal(RA.group_dest(n, [k.view(np.uint64)], [None], [False], 7), dest_rank_np(k, 7))
    z = np.array([0.0, -0.0], np.float64).view(np.uint64)
    for items, reals in (([z], [True]), ([np.array([5, 5], np.uint64), z], [False, True])):
        assert len(set(RA.group_dest(2, items, [None] * len(items), reals, 8))) == 1


def _scatter(lib, cols, nns, dest, n_parts, cap):
    """scatter_to_regions of host columns: returns (status, rows[q], overflow, regions[q][c] incl. their guards)"""
    n, nc = len(dest), len(cols)
    dev = _Dev(lib)
    regs = [[X.Buf(lib, (cap + 64) * 8) for _ in range(nc + 1)] for _ in range(n_parts)]
    try:
        dc = (_DCol * nc)(*[_DCol(dev.put(v).addr(), dev.bitmap(nn)) for v, nn in zip(cols, nns)])
        table = dev.put(np.array([regs[q][c].addr() for q in range(n_parts) for c in range(nc + 1)], np.uint64))
        d = dev.put(np.asarray(dest, np.uint8))
        rows, ovf = X.Buf(lib, 64), X.Buf(lib, 8)
        dev.bufs += [rows, ovf]
        scratch = (C.c_void_p * 6)()
        st = _scatter_to_regions(lib)(dc, nc, d.addr(), n, n_parts, table.addr(), cap, rows.addr(), ovf.addr(), C.addressof(scratch), None)
        for i in (0, 2, 4):
            if scratch[i]:
                lib.tq_device_free(C.c_void_p(scratch[i]))
        got = [[r.get() for r in rq] for rq in regs]
        return st, rows.get(np.uint32)[:n_parts], int(ovf.get()[0]), got
    finally:
        dev.free()
        for rq in regs:
            for r in rq:
                r.free()


@pytest.mark.parametrize("n_parts", [1, 2, 3])
def test_emu_scatter_to_regions(emu, n_parts):
    """every combination of region sizes from {0, 1, 63, 64, 65} per destination: each destination's rows in input order,
    column-wise, the mask word last (bit c = column c NOT NULL), rows[] exact, nothing past the rows; a cap one row short of
    the largest region: overflow = 1 and nothing written at or past the cap"""
    rng = np.random.default_rng(n_parts)
    nc = 3
    for counts in itertools.product(COUNTS, repeat=n_parts):
        n = sum(counts)
        if n == 0:
            continue
        dest = rng.permutation(np.repeat(np.arange(n_parts), counts))
        cols = [rng.integers(0, 1 << 62, n).astype(np.uint64) for _ in range(nc)]
        nns = [rng.random(n) >= 0.4, None, rng.random(n) >= 0.1]
        mask = sum((nn if nn is not None else np.ones(n, bool)).astype(np.uint64) << np.uint64(c) for c, nn in enumerate(nns))
        for cap in (max(counts), max(counts) - 1):
            if cap < 1:
                continue
            st, rows, ovf, regs = _scatter(emu, cols, nns, dest, n_parts, cap)
            assert st == L.TQ_OK
            assert list(rows) == list(counts), (counts, rows)
            assert ovf == (1 if max(counts) > cap else 0)
            for q in range(n_parts):
                idx = np.flatnonzero(dest == q)[:cap]
                for c, want in enumerate([x[idx] for x in cols] + [mask[idx]]):
                    assert np.array_equal(regs[q][c][:len(idx)], want), (counts, cap, q, c)
                    assert np.all(regs[q][c][len(idx):] == X.SENTINEL), (counts, cap, q, c, "a write past the rows or the cap")


def test_emu_scatter_wide_rows(emu):
    """63 wire columns + the mask word (the widest row): every column and every mask bit lands"""
    rng = np.random.default_rng(9)
    n, nc, n_parts = 130, 63, 2
    dest = rng.integers(0, n_parts, n)
    cols = [rng.integers(0, 1 << 62, n).astype(np.uint64) for _ in range(nc)]
    nns = [rng.random(n) >= 0.5 if c % 3 == 0 else None for c in range(nc)]
    mask = sum((nn if nn is not None else np.ones(n, bool)).astype(np.uint64) << np.uint64(c) for c, nn in enumerate(nns))
    st, rows, ovf, regs = _scatter(emu, cols, nns, dest, n_parts, n)
    assert st == L.TQ_OK and ovf == 0
    for q in range(n_parts):
        idx = np.flatnonzero(dest == q)
        assert rows[q] == len(idx)
        for c, want in enumerate([x[idx] for x in cols] + [mask[idx]]):
            assert np.array_equal(regs[q][c][:len(idx)], want)
