"""CPU suite: the key dictionaries (csrc/dict.cu KeyDict / MultiKeyEncoder, csrc/strdict.cu StringDict) run under the emulation
build (tests/emu) on inputs aimed with tests/dict_targets.py: values and strings that share one probe chain at the table's
last slot (so the chain wraps to slot 0), strings that differ only past byte 256 — including pairs with exactly the same 64-bit
hash — or only by a trailing NUL, the marker value, NULLs, sign-bit values, and batches that make the tables rehash.  Every
result is checked against a Python dict: equal key <=> equal id.  The join and aggregation trust that contract without
verifying matches (DESIGN §2), so a dictionary that broke it would return wrong rows without any error.

A probe loop that never ends is a failure too: each case runs in a forked child with a time limit."""
import ctypes as C
import multiprocessing as mp
import os
import subprocess
import traceback

import numpy as np
import pytest

import dict_targets as D

EMU_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
P = C.c_void_p


@pytest.fixture(scope="module")
def emu():
    subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
    lib = C.CDLL(os.path.join(EMU_DIR, "libtq_emu.so"))
    lib.tq_emu_sd_hash.restype = C.c_uint64
    lib.tq_emu_sd_hash.argtypes = [C.c_char_p, C.c_int64]
    lib.tq_emu_sd_new.restype = P
    lib.tq_emu_sd_free.argtypes = [P]
    lib.tq_emu_sd_encode.argtypes = [P, P, P, P, C.c_int64, C.c_int32, P, P, P]
    lib.tq_emu_mk_new.restype = P
    lib.tq_emu_mk_new.argtypes = [C.c_int32]
    lib.tq_emu_mk_free.argtypes = [P]
    lib.tq_emu_mk_encode.argtypes = [P, P, P, P, C.c_int64, C.c_int32, C.c_int32, P, P, P]
    return lib


def bounded(fn, timeout=120):
    """run fn() in a forked child: a kernel that loops forever (a probe chain that never ends) fails the test instead of hanging it"""
    ctx = mp.get_context("fork")
    rd, wr = ctx.Pipe(duplex=False)

    def child():
        try:
            fn()
            wr.send("")
        except BaseException:
            wr.send(traceback.format_exc())

    p = ctx.Process(target=child)
    p.start()
    msg = rd.recv() if rd.poll(timeout) else None
    if msg is None:
        p.kill()
        p.join()
        pytest.fail(f"the dictionary did not finish within {timeout} s (a probe chain that never ends?)")
    p.join()
    assert msg == "", msg


def _bits(words, n):
    return ((np.asarray(words, dtype=np.uint32)[np.arange(n) >> 5] >> (np.arange(n) & 31).astype(np.uint32)) & 1).astype(bool)


def _pack(not_null):
    nn = np.asarray(not_null, dtype=bool)
    w = np.zeros((len(nn) + 31) // 32 + 1, dtype=np.uint32)
    for i in np.nonzero(nn)[0]:
        w[i >> 5] |= np.uint32(1 << (i & 31))
    return w


class StrDict:
    def __init__(self, lib):
        self.lib, self.h = lib, lib.tq_emu_sd_new()

    def encode(self, cells, insert):
        """cells: list of bytes or None (NULL) -> (ids uint64, valid bool, count, n_slots)"""
        n = len(cells)
        off, data = D.cells_from_vocab([c or b"" for c in cells], np.arange(n))
        data = np.concatenate([data, np.zeros(16, np.uint8)])
        nn = np.array([c is not None for c in cells])
        bm = _pack(nn)
        ids = np.full(max(n, 1), 7, dtype=np.uint64)
        valid = np.zeros((n + 31) // 32 + 1, dtype=np.uint32)
        geom = np.zeros(2, dtype=np.uint64)
        rc = self.lib.tq_emu_sd_encode(self.h, off.ctypes.data, data.ctypes.data, bm.ctypes.data, n, int(insert), ids.ctypes.data,
                                       valid.ctypes.data, geom.ctypes.data)
        assert rc == 0
        return ids[:n], _bits(valid, n), int(geom[0]), int(geom[1])

    def close(self):
        self.lib.tq_emu_sd_free(self.h)


class KeyEncoder:
    def __init__(self, lib, k):
        self.lib, self.k, self.h = lib, k, lib.tq_emu_mk_new(k)

    def encode(self, cols, nulls, insert, null_is_value, no_signbit=None):
        """cols: k uint64 arrays; nulls: k bool arrays (True = NULL) -> (words uint64, valid bool, geometry list of (count, n_slots):
        the k column dictionaries, then the pair dictionaries)"""
        n = len(cols[0])
        cols = [np.ascontiguousarray(c, dtype=np.uint64) for c in cols]
        bms = [_pack(~np.asarray(x, dtype=bool)) for x in nulls]
        cp = (C.c_void_p * self.k)(*[c.ctypes.data for c in cols])
        bp = (C.c_void_p * self.k)(*[b.ctypes.data for b in bms])
        ns = np.array(no_signbit if no_signbit is not None else [0] * self.k, dtype=np.uint8)
        out = np.zeros(max(n, 1), dtype=np.uint64)
        bm = np.zeros((n + 31) // 32 + 1, dtype=np.uint32)
        geom = np.zeros(4 * self.k, dtype=np.uint64)
        rc = self.lib.tq_emu_mk_encode(self.h, cp, bp, ns.ctypes.data, n, int(insert), int(null_is_value), out.ctypes.data, bm.ctypes.data,
                                       geom.ctypes.data)
        assert rc == 0
        g = [(int(geom[2 * i]), int(geom[2 * i + 1])) for i in range(2 * self.k - 2)]
        return out[:n], _bits(bm, n), g

    def close(self):
        self.lib.tq_emu_mk_free(self.h)


def assert_ids_follow_keys(keys, ids, first_id):
    """equal key <=> equal id, and the ids are exactly first_id .. first_id + distinct - 1"""
    seen, back = {}, {}
    for k, i in zip(keys, ids.tolist()):
        assert seen.setdefault(k, i) == i, f"one key, two ids: {k!r}"
        assert back.setdefault(i, k) == k, f"one id {i}, two keys: {back[i]!r} / {k!r}"
    assert sorted(back) == list(range(first_id, first_id + len(back)))
    return seen


# ---------------------------------------------------------------- the restatement
def test_restated_string_hash_equals_the_library(emu):
    rng = np.random.default_rng(11)
    cells = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in range(0, 1101)]
    cells += [b"\xff" * n for n in (7, 8, 9, 255, 256, 257, 511, 512, 513)] + [b"\0" * n for n in (1, 8, 9, 256, 257)]
    cells += [rng.integers(0x80, 256, n, dtype=np.uint8).tobytes() for n in (1, 31, 32, 33, 300, 1024, 1100)]
    for c in cells:
        assert D.sd_hash(c) == emu.tq_emu_sd_hash(c, len(c)), len(c)


def test_aimers_land_where_aimed(emu):
    rng = np.random.default_rng(12)
    for length, vary_at in ((8, 0), (13, 8), (300, 0), (300, 256), (600, 296)):
        s = D.chain_strings(rng, 8, length, vary_at=vary_at)
        assert len(set(s)) == 8 and all(len(x) == length for x in s)
        for x in s:
            h = emu.tq_emu_sd_hash(x, length)
            assert h == D.sd_hash(x)
            assert all(D.sd_slot(h, 1 << b) == (1 << b) - 1 for b in range(10, 17))
    for at in (0, 256, 504):
        base = rng.integers(0, 256, 1100, dtype=np.uint8).tobytes()
        twin = D.colliding_twin(base, at)
        assert twin != base and twin[:at] == base[:at] and twin[at + 264:] == base[at + 264:]
        assert emu.tq_emu_sd_hash(twin, len(twin)) == emu.tq_emu_sd_hash(base, len(base))
    v = D.chain_values(rng, 100)
    for b in (12, 16, 20, 24):
        assert (D.kd_slot(v, 1 << b) == np.uint64((1 << b) - 1)).all()


# ---------------------------------------------------------------- KeyDict / MultiKeyEncoder
SIGN = np.uint64(1 << 63)


def test_value_dict_chain_wraps_marker_null_and_signbit(emu):
    def body():
        rng = np.random.default_rng(21)
        chain = D.chain_values(rng, 60)                       # one chain from the last slot across slot 0
        hi = chain[:40][(chain[:40] & SIGN) != 0][:5]        # present values with bit 63 set
        assert len(hi) == 5
        vals = np.concatenate([chain[:40], [D.DICT_MARKER], rng.integers(0, 1 << 62, 30, dtype=np.uint64)]).astype(np.uint64)
        idx = rng.integers(0, len(vals), 1500)
        c0 = vals[idx]
        n0 = rng.random(1500) < 0.05
        c1 = rng.integers(0, 3, 1500).astype(np.uint64)
        n1 = rng.random(1500) < 0.05
        enc = KeyEncoder(emu, 2)
        w, ok, g = enc.encode([c0, c1], [n0, n1], insert=True, null_is_value=True)
        (cnt0, slots0), (cnt1, slots1) = g[0], g[1]
        assert slots0 == D.kd_grow(0, 0, 1500) == 4096 and slots1 == 4096
        assert (D.kd_slot(chain, slots0) == np.uint64(slots0 - 1)).all()
        assert ok.all()
        id0, id1 = (w >> np.uint64(32)).astype(np.int64), (w & np.uint64(0xFFFFFFFF)).astype(np.int64)
        assert (id0[n0] == D.MK_ID_NULL).all() and (id1[n1] == D.MK_ID_NULL).all()
        is_marker = ~n0 & (c0 == np.uint64(D.DICT_MARKER))
        assert is_marker.any() and (id0[is_marker] == D.MK_ID_EMPTYVAL).all()
        reg = ~n0 & ~is_marker
        ids_of = assert_ids_follow_keys(c0[reg].tolist(), id0[reg], D.MK_FIRST_ID)
        assert cnt0 == len(ids_of)
        assert_ids_follow_keys(c1[~n1].tolist(), id1[~n1], D.MK_FIRST_ID)

        # lookup only (join probe): absent values on the same chain walk past slot n_slots - 1 to 0 and miss; present values keep
        # their ids; NULL invalidates the row; with no_signbit a value >= 2^63 never matches, even when present
        absent = chain[40:]
        pv = np.concatenate([absent, chain[:40], [D.DICT_MARKER], hi]).astype(np.uint64)
        m = len(pv)
        pn = np.zeros(m, bool)
        pn[len(absent) + 3] = True
        for no_sign in (0, 1):
            w2, ok2, g2 = enc.encode([pv, np.full(m, c1[~n1][0])], [pn, np.zeros(m, bool)], insert=False, null_is_value=False,
                                     no_signbit=[no_sign, 0])
            assert g2 == g
            for r in range(m):
                v = int(pv[r])
                if pn[r] or (v not in ids_of and v != D.DICT_MARKER) or (no_sign and v >> 63):
                    assert not ok2[r] and int(w2[r]) == D.MK_PAIR_MISS, (r, hex(v))
                else:
                    want = D.MK_ID_EMPTYVAL if v == D.DICT_MARKER else ids_of[v]
                    assert ok2[r] and int(w2[r]) >> 32 == want, (r, hex(v))
        enc.close()
    bounded(body)


def test_value_dict_ids_survive_rehashes(emu):
    def body():
        rng = np.random.default_rng(22)
        chain = D.chain_values(rng, 600)
        enc = KeyEncoder(emu, 2)
        ids_of, slots, count, sizes = {}, 0, 0, []
        batches = []
        for b, rows in enumerate((1000, 3000, 9000)):        # the table grows (a rehash) before batches 2 and 3
            fresh = rng.integers(0, 1 << 64, rows // 3, dtype=np.uint64, endpoint=False)
            pool = np.concatenate([chain[200 * b:200 * (b + 1)], fresh] + [x[0] for x in batches])
            c0 = pool[rng.integers(0, len(pool), rows)]
            c1 = np.zeros(rows, np.uint64)
            new = len(set(c0.tolist()) - set(ids_of))
            slots = D.kd_grow(slots, count, rows)
            sizes.append(slots)
            w, ok, g = enc.encode([c0, c1], [np.zeros(rows, bool)] * 2, insert=True, null_is_value=True)
            count += new
            assert g[0] == (count, slots)
            assert (D.kd_slot(chain[:200 * (b + 1)], slots) == np.uint64(slots - 1)).all()
            got = (w >> np.uint64(32)).astype(np.int64)
            for v, i in zip(c0.tolist(), got.tolist()):
                assert ids_of.setdefault(v, i) == i, hex(v)
            batches.append((c0, got))
            for pc0, pid in batches:                           # every earlier batch still encodes to the same ids
                w2, ok2, _ = enc.encode([pc0, np.zeros(len(pc0), np.uint64)], [np.zeros(len(pc0), bool)] * 2, insert=False,
                                        null_is_value=False)
                assert ok2.all() and np.array_equal((w2 >> np.uint64(32)).astype(np.int64), pid)
        assert sizes == sorted(set(sizes)) and len(sizes) == 3
        assert sorted(set(ids_of.values())) == list(range(2, 2 + count))
        enc.close()
    bounded(body)


def test_three_column_words_follow_tuples(emu):
    def body():
        rng = np.random.default_rng(23)
        chain = D.chain_values(rng, 12)
        doms = [np.concatenate([chain[:4], [D.DICT_MARKER, 5]]).astype(np.uint64),
                np.array([0, 1, D.DICT_MARKER, 1 << 63], dtype=np.uint64), chain[4:10]]
        n = 3000
        cols = [d[rng.integers(0, len(d), n)] for d in doms]
        nulls = [rng.random(n) < 0.1 for _ in range(3)]
        key = lambda r, cs, ns: tuple(None if ns[i][r] else int(cs[i][r]) for i in range(3))
        enc = KeyEncoder(emu, 3)
        w, ok, g = enc.encode(cols, nulls, insert=True, null_is_value=True)
        assert ok.all()
        tuples = [key(r, cols, nulls) for r in range(n)]
        words = {}
        back = {}
        for t, x in zip(tuples, w.tolist()):
            assert words.setdefault(t, x) == x, t
            assert back.setdefault(x, t) == t, (hex(x), back[x], t)
        assert g[3][0] == len({t[:2] for t in tuples})           # the pair dictionary holds every distinct (col0, col1)
        # join probe: every present tuple finds its word; a tuple of present values that never occurred, a NULL in any
        # column, or an absent value misses
        m = 2000
        pc = [d[rng.integers(0, len(d), m)] for d in doms]
        pc[2][:50] = chain[10]                                    # absent from column 2, on its chain
        pn = [rng.random(m) < 0.05 for _ in range(3)]
        w2, ok2, _ = enc.encode(pc, pn, insert=False, null_is_value=False)
        hits = 0
        for r in range(m):
            t = key(r, pc, pn)
            if None in t or t not in words:
                assert not ok2[r] and int(w2[r]) == D.MK_PAIR_MISS, t
            else:
                hits += 1
                assert ok2[r] and int(w2[r]) == words[t], t
        assert hits > 500 and not ok2[:50].any()
        enc.close()
    bounded(body)


# ---------------------------------------------------------------- StringDict
def _string_cases(rng):
    chain = D.chain_strings(rng, 48, 300)                       # one chain at the last slot of every table up to 2^16 slots
    twins = [D.colliding_twin(s, 0) for s in chain[:8]]         # same hash, same length, differ past byte 256 (and at byte 1)
    long_base = rng.integers(0, 256, 1100, dtype=np.uint8).tobytes()
    deep_twins = [D.colliding_twin(long_base, at) for at in (256, 512)]
    fam = []
    for off in (255, 256, 257, 511, 512):
        fam += D.differ_at(long_base[:off + 9], off, 3)
    fam += D.trailing_nuls(long_base[:256], 3) + D.trailing_nuls(b"", 3) + D.trailing_nuls(b"\x80\xff", 3)
    return chain, twins, [long_base] + deep_twins, fam


def test_string_dict_chains_collisions_and_long_families(emu):
    def body():
        rng = np.random.default_rng(31)
        chain, twins, deep, fam = _string_cases(rng)
        present = chain[:32] + twins[:4] + deep[:2] + fam
        absent = chain[32:] + twins[4:] + deep[2:] + [f + b"\0" for f in fam if len(f) == 264]
        assert not set(absent) & set(present)
        n = 700
        cells = [present[i] for i in rng.integers(0, len(present), n)]
        cells[::29] = [None] * len(cells[::29])
        sd = StrDict(emu)
        ids, valid, count, slots = sd.encode(cells, insert=True)
        assert slots == D.sd_grow(0, 0, n) == 2048
        assert all(D.sd_slot(D.sd_hash(s), slots) == slots - 1 for s in chain + twins)
        nn = np.array([c is not None for c in cells])
        assert np.array_equal(valid, nn) and (ids[~nn] == np.uint64(D.SD_ID_MISS)).all()
        ids_of = assert_ids_follow_keys([c for c in cells if c is not None], ids[nn], 0)
        assert count == len(ids_of)
        # lookup only: present strings keep their ids; absent strings on the same chain, and the colliding twins of present
        # strings, walk the chain across slot 0 and miss
        look = present + absent + [None]
        ids2, valid2, count2, slots2 = sd.encode(look, insert=False)
        assert (count2, slots2) == (count, slots)
        for s, i, ok in zip(look, ids2.tolist(), valid2.tolist()):
            if s in ids_of:
                assert ok and i == ids_of[s], s[:16]
            else:
                assert not ok and i == D.SD_ID_MISS, (None if s is None else (len(s), s[:16]))
        sd.close()
    bounded(body)


def test_string_dict_ids_survive_rehashes(emu):
    def body():
        rng = np.random.default_rng(32)
        chain = D.chain_strings(rng, 60, 40, vary_at=32)
        sd = StrDict(emu)
        ids_of, slots, count, batches, sizes = {}, 0, 0, [], []
        for b, rows in enumerate((400, 1200, 3000)):          # the table grows (a rehash) before batches 2 and 3
            words = [b"%d:%d" % (b, i) + bytes([0x80 + i % 128]) * (i % 300) for i in range(rows // 4)] + chain[20 * b:20 * (b + 1)]
            if batches:
                words += batches[-1][0][:100]
            cells = [words[i] for i in rng.integers(0, len(words), rows)]
            slots = D.sd_grow(slots, count, rows)
            sizes.append(slots)
            ids, valid, cnt, got_slots = sd.encode(cells, insert=True)
            count += len(set(cells) - set(ids_of))
            assert (cnt, got_slots) == (count, slots)
            assert all(D.sd_slot(D.sd_hash(s), slots) == slots - 1 for s in chain)
            for s, i in zip(cells, ids.tolist()):
                assert ids_of.setdefault(s, i) == i
            batches.append((cells, ids))
            for pc, pid in batches:
                ids2, valid2, _, _ = sd.encode(pc, insert=False)
                assert valid2.all() and np.array_equal(ids2, pid)
        assert sizes == sorted(set(sizes)) and len(sizes) == 3
        assert sorted(set(ids_of.values())) == list(range(count))
        sd.close()
    bounded(body)
