"""The key dictionaries on the device at their edges (csrc/dict.cu, csrc/strdict.cu), through the operators that use them:

  * string-key joins (VARCHAR alone and the reference's default {BIGINT, VARCHAR} key) whose build strings share one probe
    chain at the dictionary's last slot, with lengths 0 ... 1100, probe strings absent from the build on the same chain, and
    probe strings that differ from a build string only past byte 256 — some with exactly the same 64-bit hash;
  * a string GROUP BY over three device batches of 2^22 rows with > 10^6 distinct strings, so the dictionary grows (rehashes)
    between batches while the aggregation states hold ids of the earlier batches; host chunks and TQ_MEM_DEVICE puts;
  * a 3-column GROUP BY with > 10^6 distinct tuples (the pair dictionary) over two batches, with aimed values, the marker
    value and NULLs;
  * a 2-column device-memory join whose build side passes 2^24 rows, so KeyDict::insert runs two sub-batches.

Every aimed case first asserts, with tests/dict_targets.py, that its inputs share the last slot at every table size the run
reaches.  Expected results follow from the integer ids the columns are built from (numpy), or from the CPU oracle."""
import ctypes as C

import numpy as np
import pytest

import dict_targets as D
import oracle_py as O
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, INT64, Column, DeviceColumn, DeviceVarColumn, VarColumn, pack_not_null, tq_array
from tinysql_b200.executor import (AGG_COUNT, AGG_FIRSTROW, AGG_MAX, AGG_MIN, INNER_JOIN, LEFT_OUTER_JOIN, RIGHT_OUTER_JOIN, HashJoinExec,
                                   MockDataSource)
from util import assert_same_multiset

pytestmark = pytest.mark.gpu


def var_column(off, data, not_null=None):
    c = object.__new__(VarColumn)
    c.tp, c.length = BYTES, len(off) - 1
    c.offsets, c.data = np.ascontiguousarray(off, dtype=np.int64), np.ascontiguousarray(data, dtype=np.uint8)
    c.bitmap = None if not_null is None else pack_not_null(not_null)
    return c


def string_column(vocab, ids, not_null=None):
    return var_column(*D.cells_from_vocab(vocab, ids), not_null)


def slice_column(col, lo, hi):
    if col.tp != BYTES:
        return col.slice(lo, hi)
    nn = None if col.bitmap is None else col.not_null()[lo:hi]
    return var_column(col.offsets[lo:hi + 1] - col.offsets[lo], col.data[col.offsets[lo]:col.offsets[hi]], nn)


# ---------------------------------------------------------------- string-key joins on aimed chains
def _join_vocab(rng):
    chain = D.chain_strings(rng, 80, 300)                  # 40 in the build, 40 absent probe strings on the same chain
    lens = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in range(0, 1101)]
    bases = [rng.integers(0x80, 256, 700, dtype=np.uint8).tobytes() for _ in range(6)]
    twins = [D.colliding_twin(b, at) for b in bases for at in (256, 384)]        # same hash, differ only past byte 256
    near = [v for b in bases for off in (257, 300, 511, 640) for v in D.differ_at(b, off, 2)[1:]]
    near += [b + b"\0" for b in bases]
    build = chain[:40] + lens + bases
    absent = chain[40:] + twins + near
    assert not set(build) & set(absent) and len(set(build)) == len(build)
    return chain, build, absent


@pytest.mark.parametrize("keys", ["varchar", "bigint_varchar"])
def test_string_join_aimed_chains(lib, keys):
    rng = np.random.default_rng(71)
    chain, build, absent = _join_vocab(rng)
    vocab = build + absent
    nb, npr = 4000, 9000
    bid = np.concatenate([np.arange(len(build)), rng.integers(0, len(build), nb - len(build))])
    rng.shuffle(bid)
    pid = np.where(rng.random(npr) < 0.5, rng.integers(0, len(build), npr), len(build) + rng.integers(0, len(absent), npr))
    bnn, pnn = rng.random(nb) >= 0.03, rng.random(npr) >= 0.03
    # the build dictionary: one insert of the whole build side; every size up to 2^16 keeps the chain at the last slot
    n_slots = D.sd_grow(0, 0, nb)
    assert n_slots <= 1 << 16
    for s in chain:
        h = D.sd_hash(s)
        assert all(D.sd_slot(h, 1 << b) == (1 << b) - 1 for b in range(10, 17))
    for t, b in zip(absent[40:52], [x for x in build[-6:] for _ in (0, 1)]):
        assert D.sd_hash(t) == D.sd_hash(b) and t[:256] == b[:256] and t != b
    bk = (bid % 3).astype(np.int64)
    pk = np.where(rng.random(npr) < 0.8, pid % 3, (pid + 1) % 3).astype(np.int64)
    bcols = [Column(INT64, bk), string_column(vocab, bid, bnn), Column(INT64, np.arange(nb, dtype=np.int64))]
    pcols = [Column(INT64, np.arange(npr, dtype=np.int64) + 10**6), string_column(vocab, pid, pnn), Column(INT64, pk)]
    bkeys, pkeys = ([1], [1]) if keys == "varchar" else ([0, 1], [2, 1])
    types_b, types_p = [INT64, BYTES, INT64], [INT64, BYTES, INT64]
    for jt, oir in ((INNER_JOIN, False), (LEFT_OUTER_JOIN, False), (RIGHT_OUTER_JOIN, True)):
        inner, outer = MockDataSource(types_b, bcols, 1000), MockDataSource(types_p, pcols, 1000)
        e = HashJoinExec(outer, inner, pkeys, bkeys, jt, oir, None, 1024)
        e.Open()
        got = e.drain()
        e.Close()
        want = O.hash_join(jt, oir, types_b, bcols, types_p, pcols, bkeys, pkeys)
        assert_same_multiset(got, want)
        if jt == INNER_JOIN:
            assert got.num_rows() > npr // 4          # the join really matches (and absent strings really are probed)


# ---------------------------------------------------------------- aggregation driver (large inputs, raw result arrays)
def run_agg(lib, types, cols, group_by, funcs, device_piece=0):
    it = (C.c_int32 * len(types))(*types)
    gb = (C.c_int32 * len(group_by))(*group_by)
    fa = (L.TQAggFunc * len(funcs))(*[L.TQAggFunc(f, a) for f, a in funcs])
    d = L.TQAggDesc(len(types), it, len(group_by), gb, len(funcs), fa, 0)
    h = C.c_void_p()
    L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
    try:
        n = cols[0].length
        if device_piece:
            for lo in range(0, n, device_piece):
                dcs = [DeviceVarColumn.from_host(slice_column(c, lo, min(n, lo + device_piece))) if c.tp == BYTES
                       else DeviceColumn.from_host(slice_column(c, lo, min(n, lo + device_piece))) for c in cols]
                try:
                    L.check(lib.tq_agg_put(h, (L.TQColumn * len(dcs))(*[x.tq() for x in dcs]), L.TQ_MEM_DEVICE))
                finally:
                    for x in dcs:
                        x.free()
        else:
            L.check(lib.tq_agg_put(h, tq_array(cols), L.TQ_MEM_HOST))
        L.check(lib.tq_agg_eof(h))
        otypes = []
        for i in range(len(funcs)):
            t = C.c_int32(0)
            L.check(lib.tq_agg_output_type(h, i, C.byref(t)))
            otypes.append(t.value)
        parts = [[] for _ in funcs]
        req = 1 << 20
        while True:
            need = (C.c_int64 * len(funcs))()
            L.check(lib.tq_agg_next_bytes(h, req, need))
            out = [VarColumn.empty(BYTES, req, int(need[i])) if t == BYTES else Column.empty(t, req) for i, t in enumerate(otypes)]
            k, eof = C.c_int64(0), C.c_int32(0)
            L.check(lib.tq_agg_next(h, req, tq_array(out, req), C.byref(k), C.byref(eof)))
            k = k.value
            for i, (t, c) in enumerate(zip(otypes, out)):
                nn = c.not_null()[:k]
                if t == BYTES:
                    parts[i].append((c.offsets[:k + 1].copy(), c.data[:c.offsets[k]].copy(), nn))
                else:
                    parts[i].append((c.values[:k].copy(), nn))
            if k == 0 or eof.value:
                break
    finally:
        L.check(lib.tq_agg_destroy(h))
    res = []
    for i, t in enumerate(otypes):
        if t == BYTES:
            offs, datas, nns = [], [], []
            base = 0
            for o, dt, nn in parts[i]:
                offs.append(o[:-1] + base)
                base += int(o[-1])
                datas.append(dt)
                nns.append(nn)
            res.append((np.concatenate(offs + [np.array([base])]), np.concatenate(datas), np.concatenate(nns)))
        else:
            res.append((np.concatenate([p[0] for p in parts[i]]), np.concatenate([p[1] for p in parts[i]])))
    return res


def cells_as_bytes(off, data):
    return [data[off[i]:off[i + 1]].tobytes() for i in range(len(off) - 1)]


# ---------------------------------------------------------------- string GROUP BY across rehashes
def _group_vocab(n_groups):
    """cell g = 4-byte little-endian g + (g % 9) bytes >= 0x80: distinct for distinct g, recoverable from the first 4 bytes"""
    g = np.arange(n_groups, dtype=np.int64)
    lens = 4 + g % 9
    off = np.zeros(n_groups + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    data = np.full(off[-1], 0x80, dtype=np.uint8) + (np.repeat(g, lens) % 127).astype(np.uint8)
    head = np.repeat(off[:-1], 4) + np.tile(np.arange(4), n_groups)
    data[head] = g.astype("<u4").view(np.uint8)
    return off, data


def _arg_vocab(rng):
    """string arguments: long cells sharing a 300-byte prefix (they differ past byte 256) and short cells, all with bytes >= 0x80;
    returned sorted in Go string (unsigned byte) order, so a vocabulary index is a rank"""
    prefix = rng.integers(0x80, 256, 300, dtype=np.uint8).tobytes()
    long_ = {prefix + rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8).tobytes() for _ in range(40)}
    long_ |= {prefix[:257 + k] for k in range(0, 40, 7)}
    short = {rng.integers(0x7E, 256, int(rng.integers(0, 12)), dtype=np.uint8).tobytes() for _ in range(200)}
    short |= {prefix[:k] for k in (1, 2, 8, 9, 255, 256)}
    return sorted(long_ | short)


@pytest.fixture(scope="module")
def group_input():
    """3 * 2^22 rows over 1.5e6 distinct GROUP BY strings, one string argument column (built once for both put modes)"""
    rng = np.random.default_rng(81)
    n, n_groups = 3 * D.AGG_BATCH_ROWS, 1_500_000
    g = rng.integers(0, n_groups, n)
    v_off, v_data = _group_vocab(n_groups)
    lens = v_off[1:] - v_off[:-1]
    col0 = var_column(*D.cells_from_table(v_off, v_data, g))
    arg = _arg_vocab(rng)
    is_long = np.array([len(s) > 256 for s in arg])
    a = np.where(rng.random(n) < 0.03, rng.choice(np.nonzero(is_long)[0], n), rng.choice(np.nonzero(~is_long)[0], n))
    ann = rng.random(n) >= 0.2
    ann[g % 1000 == 7] = False                                  # some groups see only NULL arguments
    col1 = string_column(arg, a, ann)
    return n, n_groups, g, lens, col0, arg, a, ann, col1


@pytest.mark.parametrize("device", [False, True], ids=["host_chunks", "device_puts"])
def test_string_group_by_across_rehashes(lib, group_input, device):
    n, n_groups, g, lens, col0, arg, a, ann, col1 = group_input
    # the dictionary of col0 grows between batches while holding the ids of the earlier ones
    slots, count, sizes = 0, 0, []
    for lo in range(0, n, D.AGG_BATCH_ROWS):
        slots = D.sd_grow(slots, count, D.AGG_BATCH_ROWS)
        sizes.append((count, slots))
        count = len(np.unique(g[:lo + D.AGG_BATCH_ROWS]))
    assert count > 10**6 and any(c > 0 and s > sizes[i][1] for i, (c, s) in enumerate(sizes[1:]))

    funcs = [(AGG_FIRSTROW, 0), (AGG_COUNT, 1), (AGG_MAX, 1), (AGG_MIN, 1), (AGG_FIRSTROW, 1)]
    res = run_agg(lib, [BYTES, BYTES], [col0, col1], [0], funcs, D.AGG_BATCH_ROWS if device else 0)
    (k_off, k_data, k_nn), (cnt, _), mx, mn, fr = res
    m = len(k_off) - 1
    assert m == count and k_nn.all()
    assert (k_off[1:] - k_off[:-1] >= 4).all()
    got_g = k_data[np.repeat(k_off[:-1], 4) + np.tile(np.arange(4), m)].view("<u4").astype(np.int64)
    assert np.array_equal(np.sort(got_g), np.unique(g))
    assert np.array_equal(k_off[1:] - k_off[:-1], lens[got_g])

    rank = {s: i for i, s in enumerate(arg)}
    want_cnt = np.bincount(g[ann], minlength=n_groups)
    assert np.array_equal(cnt, want_cnt[got_g])
    big = len(arg)
    hi = np.full(n_groups, -1, dtype=np.int64)
    lo_ = np.full(n_groups, big, dtype=np.int64)
    np.maximum.at(hi, g[ann], a[ann])
    np.minimum.at(lo_, g[ann], a[ann])
    has = want_cnt[got_g] > 0
    for (o, dt, nn), want in ((mx, hi), (mn, lo_)):
        assert np.array_equal(nn, has)
        got = np.array([rank[c] if ok else -1 for c, ok in zip(cells_as_bytes(o, dt), nn)])
        assert np.array_equal(got[has], want[got_g][has])
    # FIRSTROW: the argument of some row of the group (NULL included)
    o, dt, nn = fr
    got = np.array([rank[c] if ok else big for c, ok in zip(cells_as_bytes(o, dt), nn)])
    pairs = np.unique(g * (big + 1) + np.where(ann, a, big))
    assert np.isin(got_g * (big + 1) + got, pairs).all()


# ---------------------------------------------------------------- multi-column keys
def test_three_column_group_by_pair_dictionary(lib):
    rng = np.random.default_rng(91)
    n = D.AGG_BATCH_ROWS + D.AGG_BATCH_ROWS // 2
    chain = D.chain_values(rng, 64)
    pools = [np.concatenate([chain, [D.DICT_MARKER]]).astype(np.uint64).view(np.int64),
             np.concatenate([np.arange(127), [D.DICT_MARKER]]).astype(np.uint64).view(np.int64),
             np.concatenate([np.arange(-128, 128), [D.DICT_MARKER]]).astype(np.uint64).view(np.int64)]
    codes, cols = [], []
    for p in pools:
        c = rng.integers(0, len(p) + 1, n)                      # code len(p) = NULL
        codes.append(c)
        nn = c < len(p)
        cols.append(Column(INT64, np.where(nn, p[np.minimum(c, len(p) - 1)], 0), nn))
    cols.append(Column(INT64, np.ones(n, dtype=np.int64)))
    tup = (codes[0] * (len(pools[1]) + 1) + codes[1]) * (len(pools[2]) + 1) + codes[2]
    want_t, want_c = np.unique(tup, return_counts=True)
    assert len(want_t) > 10**6
    # column 0: every KeyDict size the two batches reach keeps the 64 aimed values on one chain at the last slot
    slots, count = 0, 0
    for _ in range(2):
        slots = D.kd_grow(slots, count, D.AGG_BATCH_ROWS)
        assert (D.kd_slot(chain, slots) == np.uint64(slots - 1)).all()
        count = len(chain)
    funcs = [(AGG_FIRSTROW, 0), (AGG_FIRSTROW, 1), (AGG_FIRSTROW, 2), (AGG_COUNT, 3)]
    res = run_agg(lib, [INT64] * 4, cols, [0, 1, 2], funcs)
    got_codes = []
    for (v, nn), p in zip(res[:3], pools):
        order = np.argsort(p)
        pos = order[np.searchsorted(p, v, sorter=order).clip(0, len(p) - 1)]
        assert (p[pos][nn] == v[nn]).all()
        got_codes.append(np.where(nn, pos, len(p)))
    got_t = (got_codes[0] * (len(pools[1]) + 1) + got_codes[1]) * (len(pools[2]) + 1) + got_codes[2]
    order = np.argsort(got_t)
    assert np.array_equal(got_t[order], want_t)
    assert np.array_equal(res[3][0][order], want_c)


def test_two_column_device_join_past_the_insert_sub_batch(lib):
    """2^24 + 4096 unique build tuples in device memory: the column dictionaries are filled in two KeyDict::insert sub-batches.
    Checked by properties: every probe row is matched exactly once, and the build payload is a function of the key."""
    rng = np.random.default_rng(101)
    nb, npr = (1 << 24) + 4096, 1 << 21
    perm = rng.permutation(nb).astype(np.int64)
    chain = D.chain_values(rng, 16, low_bits=26).view(np.int64)   # the first sub-batch already needs 2^25 slots
    b1 = perm >> 4
    b2 = chain[perm & 15]                                       # 16 aimed values: one chain at the last slot of every table
    bv = 7 * b1 + (perm & 15) + 1
    sizes = D.kd_insert_slots(0, 0, nb, [16, 0])[2]
    assert len(sizes) == 2 and all((D.kd_slot(chain, s) == np.uint64(s - 1)).all() for s in sizes)
    rows = rng.integers(0, nb, npr)
    pk1, pk2 = b1[rows], b2[rows]
    pv = np.arange(npr, dtype=np.int64)
    dcols = [DeviceColumn.from_host(Column(INT64, x)) for x in (b1, b2, bv, pk1, pk2, pv)]
    t = (C.c_int32 * 3)(INT64, INT64, INT64)
    bk, pk = (C.c_int32 * 2)(0, 1), (C.c_int32 * 2)(0, 1)
    d = L.TQJoinDesc(INNER_JOIN, 1, 3, t, 3, t, 2, bk, pk, 0, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    try:
        barr = (L.TQColumn * 3)(*[x.tq() for x in dcols[:3]])
        parr = (L.TQColumn * 3)(*[x.tq() for x in dcols[3:]])
        for arr in (barr, parr):
            for i in range(3):
                arr[i].null_bitmap = None
        L.check(lib.tq_join_put_build(h, barr, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        L.check(lib.tq_join_put_probe(h, parr, None, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_probe_eof(h))
        got = [[] for _ in range(6)]
        while True:
            out = (L.TQColumn * 6)()
            k, eof = C.c_int64(0), C.c_int32(0)
            L.check(lib.tq_join_next_device(h, out, C.byref(k), C.byref(eof)))
            for c in range(6):
                x = np.empty(k.value, dtype=np.int64)
                if k.value:
                    L.check(lib.tq_memcpy_d2h(x.ctypes.data, out[c].data, k.value * 8))
                got[c].append(x)
            if eof.value or k.value == 0:
                break
    finally:
        L.check(lib.tq_join_destroy(h))
        for x in dcols:
            x.free()
    g1, g2, gv, q1, q2, qv = [np.concatenate(x) for x in got]
    assert len(qv) == npr and np.array_equal(np.sort(qv), pv)
    assert np.array_equal(g1, q1) and np.array_equal(g2, q2)
    slot = np.searchsorted(np.sort(chain), g2)
    assert np.array_equal(gv, 7 * g1 + np.argsort(chain)[slot] + 1)
    assert np.array_equal(q1, pk1[qv]) and np.array_equal(q2, pk2[qv])
