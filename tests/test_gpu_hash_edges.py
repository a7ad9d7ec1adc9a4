"""The hash tables' edges, reached on purpose with aimed keys (tests/hash_targets.py inverts the placement hashes).

Random keys almost never reach these paths, and a bug on them silently loses rows:
- the streaming build's hand-overs to the general build: a sub-table over the load limit, a build-scatter slab that
  overflows, and a completely full sub-table on the loop path (several sub-tables per scatter bin);
- probe chains that wrap at the end of a table (next to the empty-marker side entry) or cross a CTA slice boundary of a
  cluster-built sub-table, through every prober;
- a segmented (multi-GPU input) probe batch with skewed keys;
- the aggregation table's bucket chain that wraps past its end while the table grows (k_agg_rehash), and the shared-memory
  pre-aggregation with colliding keys.
Every test first checks, with the restated host formulas, that its input lies on the intended edge (with 10 % margin where
the edge is a count), then compares the result with the CPU oracle or checks the C3 properties on every row."""
import ctypes as C

import numpy as np
import pytest

import hash_targets as H
import oracle_py as O
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import FLOAT64, INT64, Chunk, Column, DeviceColumn, device_to_host
from tinysql_b200.executor import (AGG_AVG, AGG_COUNT, AGG_FIRSTROW, AGG_MAX, AGG_MIN, AGG_SUM, INNER_JOIN, LEFT_OUTER_JOIN,
                                   HashAggExec, HashJoinExec, MockDataSource)
from util import assert_col_equal, assert_same_multiset

pytestmark = pytest.mark.gpu

EMPTY_MARKER = np.int64(np.uint64(H.EMPTY_KEY).astype(np.int64))
PART_MAX_SMEM_BYTES = 128 << 10
JOIN_SWITCHES = ("TQ_JOIN_PART_ROWS", "TQ_JOIN_NO_FAST")


def _inside(x, lo, hi, what):
    assert x >= lo * 1.1 and x * 1.1 <= hi, f"{what}: {x} is not inside ({lo}, {hi}) with a 10 % margin"


def _switches(monkeypatch, **env):
    for k in JOIN_SWITCHES + ("TQ_AGG_NO_PREAGG", "TQ_AGG_PREAGG_PART"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _build_cols(bk, nb):
    return [Column(INT64, bk)] + [Column(INT64, bk * (c + 3) + c) for c in range(1, nb)]


def _join(lib, bcols, pcols, jt=INNER_JOIN, oir=True, chunk=1 << 20, batch=0):
    btypes, ptypes = [INT64] * len(bcols), [INT64] * len(pcols)
    e = HashJoinExec(MockDataSource(ptypes, pcols, chunk), MockDataSource(btypes, bcols, chunk), [0], [0], jt, oir, None, batch)
    e.Open()
    got = e.drain()
    st = (C.c_int64 * 8)()
    L.check(lib.tq_join_stats(e.handle, st))
    e.Close()
    assert_same_multiset(got, O.hash_join(jt, oir, btypes, bcols, ptypes, pcols, [0], [0]))
    return list(st)


def _hits_and_misses(rng, bk, aimed, misses, n_random):
    pk = np.concatenate([aimed, aimed, misses, rng.choice(bk, n_random)])
    rng.shuffle(pk)
    return [Column(INT64, pk), Column(INT64, np.arange(len(pk)))]


# ------------------------------------------------------------------ streaming-build hand-overs
@pytest.mark.parametrize("part_rows", [None, "20000"])
@pytest.mark.parametrize("nb", [2, 3])
def test_stream_build_load_limit_hands_over(lib, monkeypatch, part_rows, nb):
    """k_build_cluster: one sub-table gets ~1.3x its mean rows — over max_rows but inside its scatter slab — so flag 4 (over
    the load limit) hands the build to the general build; probed with hits and with misses aimed at that sub-table"""
    _switches(monkeypatch, **({"TQ_JOIN_PART_ROWS": part_rows} if part_rows else {}))
    rng = np.random.default_rng(nb * 10 + (part_rows is None))
    n = 1_000_000
    g = H.stream_geometry(n, nb, int(part_rows or H.PART_TARGET_ROWS))
    assert g["lbits"] == 0  # one sub-table per scatter bin: the slab bounds the sub-table
    last = (1 << g["tbits"]) - 1
    n_hot = int(1.3 * n / (1 << g["tbits"]))
    _inside(n_hot, g["max_rows"], g["bin_slab"], "rows of the aimed sub-table")
    hot = H.join_keys(rng, n_hot, last, g["tbits"], 0, 1 << 32)
    bk = np.concatenate([hot, H.join_keys_not_in_tables(rng, n - n_hot, [last], g["tbits"], exclude=hot)])
    rng.shuffle(bk)
    cnt = np.bincount(H.table_of(H.hash_key(bk), g["tbits"]).astype(np.int64), minlength=last + 1)
    assert cnt[last] == n_hot and cnt[:last].max() < g["max_rows"]  # only the aimed sub-table is over the limit
    misses = H.join_keys(rng, 20000, last, g["tbits"], 0, 1 << 32, exclude=bk)
    _join(lib, _build_cols(bk, nb), _hits_and_misses(rng, bk, hot, misses, 400_000))


def test_stream_build_scatter_slab_overflow_hands_over(lib, monkeypatch):
    """k_scatter_aos of the build side: one bin receives more rows than slab_rows(n, n_bins) — the slab overflows
    (cursor 2) and the general build answers"""
    _switches(monkeypatch)
    rng = np.random.default_rng(41)
    n = 1_000_000
    g = H.stream_geometry(n, 2)
    last = g["n_bins"] - 1
    n_hot = int(1.3 * g["bin_slab"])
    _inside(g["bin_slab"], 0, n_hot, "slab rows below the aimed bin's rows")
    hot = H.join_keys(rng, n_hot, last, g["bbits"], 0, 1 << 32)
    bk = np.concatenate([hot, H.join_keys_not_in_tables(rng, n - n_hot, [last], g["bbits"], exclude=hot)])
    rng.shuffle(bk)
    misses = H.join_keys(rng, 20000, last, g["bbits"], 0, 1 << 32, exclude=bk)
    _join(lib, _build_cols(bk, 2), _hits_and_misses(rng, bk, hot, misses, 400_000))


def _device_join(lib, bcols, pcols):
    """build + one probe batch through the device-memory C-ABI; returns (result columns, tq_join_stats)"""
    d_b, d_p = [DeviceColumn.from_host(c) for c in bcols], [DeviceColumn.from_host(c) for c in pcols]
    t = (C.c_int32 * len(bcols))(*([1] * len(bcols)))
    k = (C.c_int32 * 1)(0)
    d = L.TQJoinDesc(0, 1, len(bcols), t, len(pcols), t, 1, k, k, 0, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    try:
        barr, parr = (L.TQColumn * len(d_b))(*[x.tq() for x in d_b]), (L.TQColumn * len(d_p))(*[x.tq() for x in d_p])
        for a in (barr, parr):
            for i in range(len(a)):
                a[i].null_bitmap = None
        L.check(lib.tq_join_put_build(h, barr, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        L.check(lib.tq_join_put_probe(h, parr, None, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_probe_eof(h))
        out = (L.TQColumn * (len(bcols) + len(pcols)))()
        n, eof = C.c_int64(0), C.c_int32(0)
        cols = [[] for _ in range(len(out))]
        while True:
            L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
            if n.value == 0:
                break
            for c in range(len(out)):
                cols[c].append(device_to_host(INT64, out[c].data, None, n.value).values)
        st = (C.c_int64 * 8)()
        L.check(lib.tq_join_stats(h, st))
    finally:
        L.check(lib.tq_join_destroy(h))
        for x in d_b + d_p:
            x.free()
    return [np.concatenate(c) if c else np.zeros(0, np.int64) for c in cols], list(st)


def test_stream_build_full_subtable_on_the_loop_path(lib, monkeypatch):
    """1e7 build rows x 3 columns at the default partition size: 2 sub-tables per scatter bin (k_build_cluster's loop path).
    ~25,000 rows go into ONE sub-table of 21,248 entries (the bin stays inside its 28,512-row slab): the table fills up,
    the inserts past that hit the `probes >= cap` break, flag 4 hands over, and the general build answers.  Checked with the
    C3 properties on every row; the build time (tq_join_stats[6]) is printed — inserts into a nearly full table are slow."""
    _switches(monkeypatch)
    rng = np.random.default_rng(97)
    n, n_probe = 10_000_000, 2_000_000
    g = H.stream_geometry(n, 3)
    assert g["lbits"] == 1 and (g["cap"], g["bin_slab"]) == (21248, 28512)
    n_hot = 25_000
    _inside(n_hot, g["cap"], g["bin_slab"], "rows of the aimed sub-table (and of its bin)")
    last_sub, last_bin = (1 << g["tbits"]) - 1, g["n_bins"] - 1
    hot = H.join_keys(rng, n_hot, last_sub, g["tbits"], 0, 1 << 32)
    bk = np.concatenate([hot, H.join_keys_not_in_tables(rng, n - n_hot, [last_bin], g["bbits"], exclude=hot)])
    rng.shuffle(bk)
    assert (H.table_of(H.hash_key(bk), g["bbits"]) == np.uint64(last_bin)).sum() == n_hot  # the bin's other sub-table is empty
    pk = np.concatenate([hot, rng.choice(bk, n_probe - n_hot)])
    rng.shuffle(pk)
    with np.errstate(over="ignore"):
        bcols = [Column(INT64, bk), Column(INT64, bk * 7 + 1), Column(INT64, bk * 3 + 2)]
    cols, st = _device_join(lib, bcols, [Column(INT64, pk), Column(INT64, np.arange(n_probe))])
    print(f"\nfull sub-table hand-over: build {st[6] / 1e6:.2f} ms (tq_join_stats[6]) for {n} rows")
    b0, b1, b2, p0, p1 = cols
    assert len(b0) == n_probe
    with np.errstate(over="ignore"):
        assert np.array_equal(b1, b0 * 7 + 1) and np.array_equal(b2, b0 * 3 + 2)
    assert np.array_equal(b0, p0) and np.array_equal(np.sort(p1), np.arange(n_probe)) and np.array_equal(p0, pk[p1])


# ------------------------------------------------------------------ wrap-around and slice boundaries
CLUSTER = 48


def _wrap_keys(rng):
    """clusters of CLUSTER keys, aimed for any table geometry (top 12 hash bits: all ones = the last table, all zeros =
    table 0; low 32 bits: [2^32 - 2048, 2^32) = the last slot, [0, 2048) = slot 0, just below r << 29 = the last slot
    before CTA slice r) and absent keys with the same home slots"""
    top_ones = (1 << 12) - 1
    wins = {"last_of_last": (top_ones, (1 << 32) - 2048, 1 << 32), "last_of_first": (0, (1 << 32) - 2048, 1 << 32),
            "first_of_first": (0, 0, 2048)}
    for r in range(1, 8):
        wins[f"below_slice_{r}"] = (top_ones, (r << 29) - 1024, r << 29)
    keys, misses = {}, {}
    taken = np.zeros(0, np.int64)
    for name, (top, lo, hi) in wins.items():
        k = H.join_keys(rng, CLUSTER + 8, top, 12, lo, hi, exclude=taken)
        keys[name], misses[name] = k[:CLUSTER], k[CLUSTER:]
        taken = np.concatenate([taken, k])
    return keys, misses


def _check_homes(keys, cap, shift, n_tables):
    assert cap >= 8 * 4 * CLUSTER  # clusters of different windows do not run into each other
    pair = 2 if shift == 1 else 1
    for name, k in keys.items():
        h = H.hash_key(k)
        tbl = H.table_of(h, int(n_tables).bit_length() - 1)
        slot = H.home_slot(h, cap, shift)
        if name == "last_of_last":
            assert (tbl == n_tables - 1).all() and (slot == cap - pair).all()   # the chain wraps to slot 0 of the last table
        elif name == "last_of_first":
            assert (tbl == 0).all() and (slot == cap - pair).all()
        elif name == "first_of_first":
            assert (tbl == 0).all() and (slot == 0).all()
        else:
            r = int(name.rsplit("_", 1)[1])
            assert cap % 16 == 0 and (tbl == n_tables - 1).all() and (slot == r * cap // 8 - pair).all()


PROBERS = ["pos_16B", "pos_32B", "general_probe_on_stream_table", "generic_smem", "generic_global", "fast_smem", "fast_global",
           "one_table"]


@pytest.mark.parametrize("prober", PROBERS)
def test_probe_chains_wrap_and_cross_slices(lib, monkeypatch, prober):
    """chains of CLUSTER keys that wrap at the end of the last table (next to the empty-marker side entry), wrap from the
    last slot of table 0 into a cluster at its slot 0, and cross every CTA slice boundary; every clustered key is probed
    (hits) and so are absent keys with the same home slots (misses that walk the whole chain).  Probers: k_probe_pos on
    a stream-built table (16- and 32-byte entries); the general partitioned probe on a stream-built table (left outer join,
    nullable probe key); the generic (TQ_JOIN_NO_FAST=1) and the fast (k_probe_part_fast, after a skewed batch has turned
    the optimistic scatter off) partitioned kernels on a general-built table, with the table image in shared memory
    (2400 rows per partition) and in global memory; the one-table k_probe (build side below 2^18 rows).  The general-built
    tables hold an empty-marker build row, so the side entry sits right after the last partition."""
    rng = np.random.default_rng(PROBERS.index(prober) + 300)
    keys, misses = _wrap_keys(rng)
    aimed = np.concatenate(list(keys.values()))
    absent = np.concatenate(list(misses.values()))
    nb = 3 if prober == "pos_32B" else 2
    general = prober.startswith(("generic", "fast")) or prober == "one_table"
    n = 100_000 if prober == "one_table" else 300_000
    part_rows = 2400 if prober.endswith("smem") else H.PART_TARGET_ROWS
    env = {}
    if prober.startswith("generic"):
        env["TQ_JOIN_NO_FAST"] = "1"
    if part_rows != H.PART_TARGET_ROWS:
        env["TQ_JOIN_PART_ROWS"] = str(part_rows)
    _switches(monkeypatch, **env)
    bg = H.join_keys_not_in_tables(rng, n - len(aimed) - 1, [], 1, exclude=np.concatenate([aimed, absent]))
    bk = np.concatenate([aimed, bg] + ([[EMPTY_MARKER]] if general else []))
    rng.shuffle(bk)
    if general:
        g = H.general_geometry(bk, nb, part_rows)
        _check_homes(keys, g["cap"], g["shift"], 1 << g["pbits"])
        image = (g["cap"] << g["shift"]) * 8
        if prober == "one_table":
            assert g["pbits"] == 0 and n < H.PART_MIN_BUILD_ROWS
        elif prober.endswith("smem"):
            assert g["pbits"] > 0 and image <= PART_MAX_SMEM_BYTES
        else:
            assert g["pbits"] > 0 and image > PART_MAX_SMEM_BYTES
    else:
        g = H.stream_geometry(len(bk), nb)
        _check_homes(keys, g["cap"], g["shift"], 1 << g["tbits"])
        cnt = np.bincount(H.table_of(H.hash_key(bk), g["tbits"]).astype(np.int64))
        assert cnt.max() <= g["max_rows"]  # unique keys, no marker, no sub-table over the limit: the streaming build keeps it
    hits = np.concatenate([aimed] * 2 + ([[EMPTY_MARKER] * 3] if general else []))  # (a probe key equal to the marker: the side entry)
    pcols = _hits_and_misses(rng, bk, hits, np.concatenate([absent] * 4), 100_000)
    bcols = _build_cols(bk, nb)
    if prober == "general_probe_on_stream_table":
        nn = rng.random(len(pcols[0].values)) > 0.05
        _join(lib, bcols, [Column(INT64, pcols[0].values, nn), pcols[1]], LEFT_OUTER_JOIN, False)
    elif prober.startswith("fast"):
        # a first batch of 2^20 rows with one hot key overflows its optimistic slab: later batches take the exact histogram
        # path, where an inner join on unique build keys runs k_probe_part_fast
        skew = rng.choice(bk, 1 << 20)
        skew[rng.random(1 << 20) < 0.8] = bg[7]
        pk = np.concatenate([skew, pcols[0].values])
        _join(lib, bcols, [Column(INT64, pk), Column(INT64, np.arange(len(pk)))], chunk=1 << 20, batch=1 << 20)
    else:
        _join(lib, bcols, pcols)


# ------------------------------------------------------------------ skewed segmented probe batch
def _dev(a):
    p = C.c_void_p()
    L.check(L.load().tq_device_alloc(max(a.nbytes, 8), C.byref(p)))
    if a.nbytes:
        L.check(L.load().tq_memcpy_h2d(p, a.ctypes.data, a.nbytes))
    return p


def test_skewed_segmented_probe_batch(lib, monkeypatch):
    """tq_join_put_probe_segments over 3 device regions with device-resident counts, ~80 % of the probe rows carrying one
    key: the batch overflows a partition slab, is gathered and re-run on the exact histogram path.  Then an ordinary skewed
    batch (which turns the optimistic scatter off) and another segmented batch on the same handle, which must be accepted.
    The whole result equals the oracle's."""
    _switches(monkeypatch)
    rng = np.random.default_rng(1234)
    nb = 1_000_000
    bk = rng.permutation(nb).astype(np.int64)
    bcols = [Column(INT64, bk), Column(INT64, bk * 7 + 1)]
    batches, next_id = [], 0

    def rows(n, hot):
        nonlocal next_id
        k = rng.integers(0, nb + nb // 10, n).astype(np.int64)   # ~9 % misses
        if hot:
            k[rng.random(n) < 0.8] = 4242
        ids = np.arange(next_id, next_id + n, dtype=np.int64)
        next_id += n
        return k, ids
    allocs = []
    t = (C.c_int32 * 2)(1, 1)
    kk = (C.c_int32 * 1)(0)
    d = L.TQJoinDesc(0, 1, 2, t, 2, t, 1, kk, kk, 0, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    d_b = [DeviceColumn.from_host(c) for c in bcols]
    out_cols = [[] for _ in range(4)]
    out = (L.TQColumn * 4)()
    n, eof = C.c_int64(0), C.c_int32(0)

    def drain():
        while True:
            L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
            if n.value == 0:
                return
            for c in range(4):
                out_cols[c].append(device_to_host(INT64, out[c].data, None, n.value).values)

    def put_segments(counts, cap, hot):
        cols = (L.TQColumn * (2 * len(counts)))()
        cnt_ptrs = (C.c_void_p * len(counts))()
        for g, m in enumerate(counts):
            k, ids = rows(m, hot)
            batches.append((k, ids))
            for c, a in enumerate((k, ids)):
                region = np.zeros(cap, np.int64)
                region[:m] = a
                p = _dev(region)
                allocs.append(p)
                cols[2 * g + c].data, cols[2 * g + c].length = p.value, m
            cp = _dev(np.array([m], np.uint64))
            allocs.append(cp)
            cnt_ptrs[g] = cp.value
        return lib.tq_join_put_probe_segments(h, len(counts), cols, cnt_ptrs, cap)
    try:
        barr = (L.TQColumn * 2)(d_b[0].tq(), d_b[1].tq())
        for i in range(2):
            barr[i].null_bitmap = None
        L.check(lib.tq_join_put_build(h, barr, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        st = (C.c_int64 * 8)()
        L.check(lib.tq_join_stats(h, st))
        P = st[2]
        counts, cap = [170_000, 200_000, 110_000], 200_000
        seg_rows = len(counts) * cap   # (at least: the regions are padded to whole scatter tiles)
        hot_rows = 0.8 * sum(counts)
        _inside(H.slab_rows(seg_rows + 3 * 8192, P, True), 0, hot_rows, "optimistic slab below the hot partition's rows")
        L.check(put_segments(counts, cap, True))
        # an ordinary skewed batch: its overflow turns the optimistic scatter off for ordinary batches
        k, ids = rows(600_000, True)
        batches.append((k, ids))
        dk, di = DeviceColumn.from_host(Column(INT64, k)), DeviceColumn.from_host(Column(INT64, ids))
        parr = (L.TQColumn * 2)(dk.tq(), di.tq())
        for i in range(2):
            parr[i].null_bitmap = None
        L.check(lib.tq_join_put_probe(h, parr, None, L.TQ_MEM_DEVICE))
        drain()
        L.check(put_segments([90_000, 150_000], 160_000, False))   # a later segmented batch is still accepted
        drain()
        L.check(put_segments([120_000, 30_000, 125_000], 125_000, True))
        L.check(lib.tq_join_probe_eof(h))
        drain()
        dk.free()
        di.free()
    finally:
        L.check(lib.tq_join_destroy(h))
        for p in allocs:
            lib.tq_device_free(p)
        for x in d_b:
            x.free()
    got = Chunk([Column(INT64, np.concatenate(c)) for c in out_cols])
    pk = np.concatenate([b[0] for b in batches])
    pv = np.concatenate([b[1] for b in batches])
    want = O.hash_join(INNER_JOIN, True, [INT64, INT64], bcols, [INT64, INT64], [Column(INT64, pk), Column(INT64, pv)], [0], [0])
    assert_same_multiset(got, want)


# ------------------------------------------------------------------ per-handle switches
def test_join_partition_size_switch_is_per_handle(lib, monkeypatch):
    """TQ_JOIN_PART_ROWS is read by each tq_join_create: unset again means the default 150,000 rows per partition"""
    rng = np.random.default_rng(2)
    bk = rng.permutation(1_000_000).astype(np.int64)
    bcols = [Column(INT64, bk), Column(INT64, bk * 7 + 1)]
    pcols = [Column(INT64, bk[:1000]), Column(INT64, np.arange(1000))]
    _switches(monkeypatch, TQ_JOIN_PART_ROWS="2400")
    assert _device_join(lib, bcols, pcols)[1][2] == 512
    _switches(monkeypatch)
    assert _device_join(lib, bcols, pcols)[1][2] == 8


# ------------------------------------------------------------------ aggregation table
CHAIN = 1500


def _agg(lib, monkeypatch, types, batches, funcs, est, not_null=(), env=None):
    """HashAggExec whose input arrives as device batches (one update call each); returns (result chunk, tq_agg_stats)"""
    _switches(monkeypatch, **(env or {}))
    e = HashAggExec(MockDataSource(types, [Column(t, np.zeros(0)) for t in types]), [0], funcs, est, not_null_cols=not_null)
    e.Open()
    for cols in batches:
        d = [DeviceColumn.from_host(c) for c in cols]
        L.check(lib.tq_agg_put(e.handle, (L.TQColumn * len(d))(*[x.tq() for x in d]), L.TQ_MEM_DEVICE))
        for x in d:
            x.free()
    got = e.drain()
    st = (C.c_int64 * 4)()
    L.check(lib.tq_agg_stats(e.handle, st))
    e.Close()
    return got, list(st)


def _check_agg(got, types, batches, funcs):
    cols = [Column(t, np.concatenate([b[i].values for b in batches]), np.concatenate([b[i].not_null() for b in batches]))
            for i, t in enumerate(types)]
    rc, want = O.hash_agg(types, cols, [0], funcs, 2)
    assert rc == 0 and got.num_rows() == want.num_rows()
    ki = [f for f, _ in funcs].index(AGG_FIRSTROW)
    for a, b in zip(_by_key(got, ki), _by_key(want, ki)):
        assert_col_equal(a, b)


def _by_key(chunk, ki):
    nn = chunk.cols[ki].not_null()
    raw = chunk.cols[ki].raw().copy()
    raw[~nn] = 0
    order = np.lexsort((raw, nn))
    return [Column(c.tp, c.values[order], c.not_null()[order]) for c in chunk.cols]


def _chain_keys(rng):
    """CHAIN keys whose mix64 shares the low 24 bits 0xFFFFFF: one bucket chain that starts at the last bucket and wraps
    past the end, for every table size up to 2^24 slots"""
    k = H.agg_keys(rng, CHAIN, 24, (1 << 24) - 1)
    for slots in (1 << 16, 1 << 18, 1 << 24):
        assert ((H.mix64(k) & np.uint64(slots - 1)) & ~np.uint64(3) == np.uint64(slots - 4)).all()
    return k


@pytest.mark.parametrize("not_null", [False, True])
def test_agg_wrapping_chain_survives_growth(lib, monkeypatch, not_null):
    """est_groups=1: the table starts at 2^16 slots with the wrapping chain in it; the second batch brings more groups than
    the load limit allows, so the table grows (k_agg_rehash moves the chain) and the deferred rows are replayed.  Generic
    update with NULL keys and NULL arguments, and the NOT NULL integer key with dyadic doubles.  Bit-exact vs the oracle."""
    rng = np.random.default_rng(55 + not_null)
    chain = _chain_keys(rng)
    fill = rng.integers(-(1 << 62), 1 << 62, 50_000)
    fill = np.unique(fill[~np.isin(fill, chain)])[:40_000]
    _inside(CHAIN + len(fill), (1 << 16) // 2, (1 << 18) // 2, "groups vs the load limits of the 2^16 and 2^18 tables")
    types = [INT64, INT64, FLOAT64]

    def batch(keys, reps):
        k = np.repeat(keys, reps)
        rng.shuffle(k)
        m = len(k)
        v = rng.integers(-1000, 1000, m)
        x = np.floor(rng.random(m) * 4096) / 16
        if not_null:
            return [Column(INT64, k), Column(INT64, v), Column(FLOAT64, x)]
        return [Column(INT64, k, rng.random(m) > 0.01), Column(INT64, v, rng.random(m) > 0.1), Column(FLOAT64, x, rng.random(m) > 0.1)]
    batches = [batch(chain, 4), batch(np.concatenate([fill, chain]), 3)]
    funcs = [(AGG_COUNT, -1), (AGG_COUNT, 1), (AGG_SUM, 1), (AGG_AVG, 1), (AGG_MAX, 1), (AGG_MIN, 1), (AGG_SUM, 2), (AGG_MIN, 2),
             (AGG_FIRSTROW, 0)]
    got, _ = _agg(lib, monkeypatch, types, batches, funcs, 1, (0, 1, 2) if not_null else ())
    _check_agg(got, types, batches, funcs)


def test_agg_preaggregation_with_colliding_chain_keys(lib, monkeypatch):
    """one batch of 2^20+ rows over the chain keys takes the shared-memory pre-aggregation (k_agg_preagg: the keys also
    collide in its per-CTA table, whose index bits 20..23 they share) and its merge into the wrapping chain; a handle
    created with TQ_AGG_NO_PREAGG=1 in the same process takes the general path — the switch is read per handle"""
    rng = np.random.default_rng(77)
    chain = _chain_keys(rng)
    assert len(np.unique((H.mix64(chain) >> np.uint64(20)) & np.uint64(4095))) < CHAIN  # collisions in the pre-aggregation table
    n = (1 << 20) + 4096
    k = chain[rng.integers(0, CHAIN, n)]
    types = [INT64, FLOAT64, FLOAT64]
    batches = [[Column(INT64, k), Column(FLOAT64, np.floor(rng.random(n) * 4096) / 16), Column(FLOAT64, np.floor(rng.random(n) * 1024) / 4)]]
    funcs = [(AGG_COUNT, -1), (AGG_SUM, 1), (AGG_AVG, 2), (AGG_COUNT, 1), (AGG_FIRSTROW, 0)]
    launches = {}
    for env in ({"TQ_AGG_NO_PREAGG": "1"}, {}, {"TQ_AGG_NO_PREAGG": "1"}):
        got, st = _agg(lib, monkeypatch, types, batches, funcs, 1, (0, 1, 2), env)
        _check_agg(got, types, batches, funcs)
        launches.setdefault(bool(env), set()).add(st[3])
    # one launch set per path; the pre-aggregated handle runs k_agg_preagg on top of the (merge) update and the collect
    assert len(launches[True]) == 1 and launches[False] == {next(iter(launches[True])) + 1}
