"""CPU suite: the string half of the GROUP BY push (csrc/partition.cu) under the emulation build of tests/emu.

- The destination of a partial row with string items (group_dest with content hashes) against the Python twin
  (tests/region_agg_ref.py) fed the dictionary's hash words (tests/dict_targets.sd_hash); "" and NULL are different words.
- The var-len scatter (scatter_to_regions_var): each region's var-len column reads back as a chunk.Column — offsets from 0
  and the cells in source order — at region ends of 0, 1, 63, 64 and 65 rows, with cells of 0 .. 4096 bytes across the
  16-byte copy chunks and the warp's 512-byte stride, NULL next to "".  A byte cap that fits the largest region exactly
  writes everything; one byte short overflows and leaves the guard bytes past the cap untouched."""
import ctypes as C
import itertools

import numpy as np
import pytest

import dict_targets as D
import exchange_ref as X
import region_agg_ref as RA
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)
from test_emu_region_agg import _DCol, _Dev
from tinysql_b200 import _lib as L

COUNTS = [0, 1, 63, 64, 65]
LENS = [0, 1, 7, 8, 9, 15, 16, 17, 255, 256, 257, 4096]
GUARD = 64


class _RegionVar(C.Structure):
    """tq::RegionVar (csrc/scatter.cuh)"""
    _fields_ = [("col", C.c_int), ("off", C.c_void_p), ("bytes", C.c_void_p), ("byte_cap", C.c_uint64)]


def _group_dest_hashed(lib):
    """tq::group_dest with per-item hash tables (csrc/scatter.cuh), by its C++ symbol"""
    fn = getattr(lib, "_ZN2tq10group_destEPKNS_4DColEPKPKmijliPhPv")
    fn.restype = C.c_int32
    fn.argtypes = [C.POINTER(_DCol), C.c_void_p, C.c_int, C.c_uint32, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
    return fn


def _scatter_var(lib):
    """tq::scatter_to_regions_var (csrc/scatter.cuh); its RegionScratch is six DevBufs {void *p; size_t cap}"""
    fn = getattr(lib, "_ZN2tq22scatter_to_regions_varEPKNS_4DColEiPKNS_9RegionVarEiPKhliPKPmlPjPyRNS_13RegionScratchEPv")
    fn.restype = C.c_int32
    fn.argtypes = [C.POINTER(_DCol), C.c_int, C.POINTER(_RegionVar), C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


def _arena(strings):
    """a dictionary arena of the strings: (offsets, bytes); id i = strings[i]"""
    off = np.zeros(len(strings) + 1, np.int64)
    np.cumsum([len(x) for x in strings], out=off[1:])
    return off, np.frombuffer(b"".join(strings) + b"\0" * 16, np.uint8).copy()


def _strings(rng, k):
    return [b""] + [rng.integers(0, 256, LENS[i % len(LENS)], dtype=np.uint8).tobytes() for i in range(1, k)]


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1000])
def test_emu_group_dest_strings_match_twin(emu, n):
    """string items route by their dictionary hash word, alone and next to INT64 / REAL items, NULLs included: k_group_dest ==
    the twin over the sd_hash words; "" and NULL get different words"""
    rng = np.random.default_rng(n)
    strings = _strings(rng, 40)
    hashes = D.sd_hashes(strings)
    assert D.sd_hash(b"") != int(RA.GROUP_NULL_WORD)
    fn = _group_dest_hashed(emu)
    for kinds in (("s",), ("s", "i"), ("i", "s"), ("s", "r", "s")):
        dev = _Dev(emu)
        try:
            vals, nns, items, twin, reals = [], [], [], [], []
            for g, k in enumerate(kinds):
                if k == "s":
                    ids = rng.integers(0, len(strings), n).astype(np.uint64)
                    vals.append(ids)
                    twin.append(hashes[ids.astype(np.int64)])
                elif k == "r":
                    v = rng.choice(np.array([0.0, -0.0, 2.5], np.float64), n).view(np.uint64)
                    vals.append(v)
                    twin.append(v)
                else:
                    v = rng.integers(-5, 5, n).astype(np.int64).view(np.uint64)
                    vals.append(v)
                    twin.append(v)
                reals.append(k == "r")
                nns.append(rng.random(n) >= 0.25 if g % 2 == 0 else None)
            items = (_DCol * len(kinds))(*[_DCol(dev.put(v).addr(), dev.bitmap(nn)) for v, nn in zip(vals, nns)])
            htab = dev.put(hashes)
            hp = (C.c_void_p * len(kinds))(*[htab.addr() if k == "s" else None for k in kinds])
            real_mask = sum(1 << g for g, r in enumerate(reals) if r)
            for n_parts in (1, 2, 3, 8):
                out = X.Buf(emu, n + 64)
                try:
                    assert fn(items, C.addressof(hp), len(kinds), real_mask, n, n_parts, out.addr(), None) == L.TQ_OK
                    got = out.get(np.uint8)
                    want = RA.group_dest(n, twin, nns, reals, n_parts)
                    assert np.array_equal(got[:n], want.astype(np.uint8)), (kinds, n_parts)
                    assert np.all(got[n:] == X.SENTINEL_BYTE)
                finally:
                    out.free()
        finally:
            dev.free()


def _scatter(lib, cols, nns, var, arenas, dest, n_parts, cap, byte_caps):
    """scatter_to_regions_var of host columns; var: the var-len wire columns, arenas: their (offsets, bytes).  Returns
    (status, rows[q], overflow, word areas [q][c] and byte areas [q][v], each with its guard)"""
    n, nc, nv = len(dest), len(cols), len(var)
    dev = _Dev(lib)
    words = [[X.Buf(lib, (cap + 1 + GUARD) * 8) for _ in range(nc + 1)] for _ in range(n_parts)]
    areas = [[X.Buf(lib, byte_caps[v] + GUARD) for v in range(nv)] for _ in range(n_parts)]
    try:
        dc = (_DCol * nc)(*[_DCol(dev.put(v).addr(), dev.bitmap(nn)) for v, nn in zip(cols, nns)])
        rv = (_RegionVar * nv)(*[_RegionVar(c, dev.put(off).addr(), dev.put(b).addr(), byte_caps[v]) for v, (c, (off, b)) in enumerate(zip(var, arenas))])
        table = dev.put(np.array([w.addr() for q in range(n_parts) for w in words[q] + areas[q]], np.uint64))
        d = dev.put(np.asarray(dest, np.uint8))
        rows, ovf = X.Buf(lib, 64), X.Buf(lib, 8)
        dev.bufs += [rows, ovf]
        L.check(lib.tq_memset_device(C.c_void_p(ovf.addr()), 0, 8))
        scratch = (C.c_void_p * 12)()
        st = _scatter_var(lib)(dc, nc, rv, nv, d.addr(), n, n_parts, table.addr(), cap, rows.addr(), ovf.addr(), C.addressof(scratch), None)
        for i in range(0, 12, 2):
            if scratch[i]:
                lib.tq_device_free(C.c_void_p(scratch[i]))
        return (st, rows.get(np.uint32)[:n_parts], int(ovf.get()[0]), [[w.get() for w in wq] for wq in words],
                [[a.get(np.uint8) for a in aq] for aq in areas])
    finally:
        dev.free()
        for wq in words:
            for w in wq:
                w.free()
        for aq in areas:
            for a in aq:
                a.free()


def _case(rng, counts, n_parts):
    """rows for the region sizes `counts`: wire columns (s ids, x, t ids) with NULLs in s next to "" cells"""
    n = sum(counts)
    dest = rng.permutation(np.repeat(np.arange(n_parts), counts))
    sa, ta = _strings(rng, 25), _strings(rng, 13)
    s = rng.integers(0, len(sa), n).astype(np.uint64)
    s[::5] = 0                                               # "" ...
    snn = np.ones(n, bool)
    snn[1::5] = False                                        # ... next to NULL
    t = rng.integers(0, len(ta), n).astype(np.uint64)
    x = rng.integers(0, 1 << 62, n).astype(np.uint64)
    return dest, [s, x, t], [snn, None, rng.random(n) >= 0.2], [sa, ta]


def _cells(strings, ids, nn):
    return [strings[int(i)] if ok else b"" for i, ok in zip(ids, nn)]


@pytest.mark.parametrize("n_parts", [1, 2, 3])
def test_emu_scatter_var_regions(emu, n_parts):
    """region sizes from {0, 1, 63, 64, 65} per destination: the 8-byte column and mask word as scatter_to_regions writes them,
    each var-len column's offsets area = its region's chunk.Column offsets (cells in source order, NULL empty) and its byte
    area = the cells; nothing past the rows + 1 offsets or the region's bytes; byte cap exact, then one byte short"""
    rng = np.random.default_rng(50 + n_parts)
    combos = list(itertools.product(COUNTS, repeat=n_parts))
    if len(combos) > 40:
        combos = [combos[i] for i in rng.choice(len(combos), 40, replace=False)]
    var = [0, 2]
    for counts in combos:
        n = sum(counts)
        if n == 0:
            continue
        dest, cols, nns, strs = _case(rng, counts, n_parts)
        arenas = [_arena(x) for x in strs]
        nn_all = [nn if nn is not None else np.ones(n, bool) for nn in nns]
        mask = sum(nn.astype(np.uint64) << np.uint64(c) for c, nn in enumerate(nn_all))
        want_cells = [[_cells(strs[v], cols[c][dest == q], nn_all[c][dest == q]) for v, c in enumerate(var)] for q in range(n_parts)]
        need = [max([sum(len(x) for x in want_cells[q][v]) for q in range(n_parts)] + [1]) for v in range(len(var))]
        cap = max(counts)
        for short in (None, 0, 1):
            caps = list(need)
            if short is not None:
                caps[short] -= 1
                if caps[short] < 1:
                    continue
            st, rows, ovf, words, areas = _scatter(emu, cols, nns, var, arenas, dest, n_parts, cap, caps)
            assert st == L.TQ_OK
            assert list(rows) == list(counts)
            assert ovf == (0 if short is None else 1), (counts, short)
            for q in range(n_parts):
                k = counts[q]
                idx = np.flatnonzero(dest == q)
                assert np.array_equal(words[q][1][:k], cols[1][idx]) and np.all(words[q][1][k:] == X.SENTINEL)
                assert np.array_equal(words[q][3][:k], mask[idx]) and np.all(words[q][3][k:] == X.SENTINEL)
                for v, c in enumerate(var):
                    cells = want_cells[q][v]
                    total = sum(len(x) for x in cells)
                    assert np.all(areas[q][v][caps[v]:] == X.SENTINEL_BYTE), (counts, short, q, v, "a byte past the cap")
                    if short is not None and total > caps[v]:
                        assert np.all(areas[q][v] == X.SENTINEL_BYTE), "an overflowed byte area got cells"
                        continue
                    off = np.zeros(k + 1, np.int64)
                    np.cumsum([len(x) for x in cells], out=off[1:])
                    assert np.array_equal(words[q][c][:k + 1].view(np.int64), off), (counts, q, v)
                    assert np.all(words[q][c][k + 1:] == X.SENTINEL), "a write past the offsets"
                    assert areas[q][v][:total].tobytes() == b"".join(cells), (counts, q, v)
                    assert np.all(areas[q][v][total:] == X.SENTINEL_BYTE), "a write past the region's cells"


def test_emu_scatter_var_every_length(emu):
    """one destination, one cell of every length in LENS at every start offset mod 16 (the cells before it vary its byte
    position), NULL next to "": the byte area is the concatenation"""
    rng = np.random.default_rng(3)
    strings = [b""] + [rng.integers(0, 256, ln, dtype=np.uint8).tobytes() for ln in LENS] + [b"x" * k for k in range(1, 16)]
    ids, nn = [], []
    for shift in range(16):
        for i in range(1, len(LENS) + 1):
            if shift:
                ids.append(len(LENS) + shift)                # a cell of `shift` bytes moves the next cell's start
                nn.append(True)
            ids += [i, 0, 0]
            nn += [True, False, True]
    ids = np.array(ids, np.uint64)
    nn = np.array(nn)
    n = len(ids)
    cells = _cells(strings, ids, nn)
    total = sum(len(x) for x in cells)
    for n_parts in (1, 2):
        dest = np.zeros(n, np.uint8) if n_parts == 1 else (np.arange(n) % 2).astype(np.uint8)
        caps = [max(sum(len(c) for c, d in zip(cells, dest) if d == q) for q in range(n_parts))]
        st, rows, ovf, words, areas = _scatter(emu, [ids], [nn], [0], [_arena(strings)], dest, n_parts, n, caps)
        assert st == L.TQ_OK and ovf == 0
        for q in range(n_parts):
            sel = [c for c, d in zip(cells, dest) if d == q]
            assert rows[q] == len(sel)
            assert areas[q][0][:sum(len(x) for x in sel)].tobytes() == b"".join(sel)
        if n_parts == 1:
            assert rows[0] == n and areas[0][0][:total].tobytes() == b"".join(cells)
