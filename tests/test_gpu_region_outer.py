"""Outer joins and nullable columns across GPUs on one GPU, every rank emulated in this process (tests/region_outer_ref.py):
tq_partition_push_regions -> published slots -> tq_region_gather -> an ordinary join handle per destination.

Per destination: every matched row's probe key has dest_rank_np(key) == destination; a probe row that cannot match (NULL key
or selected == 0) of an outer join comes out once, as its miss row, on the rank that held it.  Over all destinations the rows
are exactly oracle_py.hash_join over every shard.  A cap one row short fails the receiving gather, which writes nothing;
a side wider than the push's 4 words is refused before anything is pushed."""
import numpy as np
import pytest

import exchange_ref as X
import oracle_py as O
import region_outer_ref as R
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import FLOAT64, INT64, UINT64, Chunk, Column
from tinysql_b200.dist import dest_rank_np
from util import assert_same_multiset

pytestmark = pytest.mark.gpu

DEFAULT_ID = -424242          # the build-id column of a defaultInner miss row: no build row has a negative id
JOINS = [(0, True), (0, False), (1, False), (2, True)]   # (join_type, outer_is_right)


def _nulls_on_edges(rng, n, p):
    """NOT-NULL bools with NULLs at every 64-row group's first and last row, and random ones"""
    nn = rng.random(n) >= p
    idx = np.arange(n)
    nn[(idx % 64 == 0) | (idx % 64 == 63)] = False
    return nn


def _shards(rng, W, sizes, key_pool, first_id, nullable, key_null_p, key_type=INT64):
    """per source ([key, id, payload], nns): keys drawn from key_pool, ids globally unique from first_id"""
    out, nid = [], first_id
    for s, n in enumerate(sizes):
        k = rng.choice(key_pool, n) if n else np.zeros(0, np.uint64)
        ids = np.arange(nid, nid + n, dtype=np.int64)
        nid += n
        pay = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
        nns = [None, None, None]
        if nullable:
            nns[0] = rng.random(n) >= key_null_p
            nns[2] = _nulls_on_edges(rng, n, 0.2)
            nns[1] = np.ones(n, bool)           # a bitmap that says NOT NULL everywhere
        out.append(([np.asarray(k).view(np.uint64), ids.view(np.uint64), pay.view(np.uint64)], nns))
    return out


def _all(shards, ci, tp):
    v = np.concatenate([cols[ci] for cols, _ in shards]) if shards else np.zeros(0, np.uint64)
    nns = [nns[ci] if nns[ci] is not None else np.ones(len(cols[0]), bool) for cols, nns in shards]
    return Column(tp, v.view({INT64: np.int64, UINT64: np.uint64, FLOAT64: np.float64}[tp]), np.concatenate(nns) if nns else None)


def _check(W, jt, oir, btypes, ptypes, bsh, psh, psel, default_inner, results):
    outer = jt != 0
    n_b, n_p = len(btypes), len(ptypes)
    # probe row id -> holding rank, and which rows cannot match
    holder, unmatchable = {}, set()
    for s, (cols, nns) in enumerate(psh):
        ids = cols[1].view(np.int64)
        d = R.routed(cols[0], nns[0], psel[s] if psel else None, W)
        for i, r in zip(ids, d):
            holder[int(i)] = s
            if r < 0:
                unmatchable.add(int(i))
    pb, bb = (n_b, 0) if oir else (0, n_p)       # first probe / build column in the output
    for d, res in enumerate(results):
        assert isinstance(res, Chunk), f"destination {d} failed with status {res}"
        if not res.num_rows():
            continue
        pkey, pid = res.cols[pb], res.cols[pb + 1].values.astype(np.int64)
        bid = res.cols[bb + 1]
        matched = bid.not_null() & (bid.values.view(np.int64) != DEFAULT_ID)
        if matched.any():
            assert np.all(dest_rank_np(pkey.raw()[matched].view(np.int64), W) == d), f"destination {d}: a pair joined on the wrong rank"
        for i in pid[~matched]:
            if int(i) in unmatchable:
                assert holder[int(i)] == d, f"miss row of probe row {i} emitted on {d}, held by {holder[int(i)]}"
        if outer:
            miss_ids = pid[~matched]
            assert len(np.unique(miss_ids)) == len(miss_ids), "a probe row came out twice as a miss row"
    bcols = [_all(bsh, c, btypes[c]) for c in range(n_b)]
    pcols = [_all(psh, c, ptypes[c]) for c in range(n_p)]
    sel = np.concatenate(psel).astype(np.uint8) if psel else None
    want = O.hash_join(jt, oir, btypes, bcols, ptypes, pcols, [0], [0], selected=sel, default_inner=default_inner)
    out_types = (list(btypes) + list(ptypes)) if oir else (list(ptypes) + list(btypes))
    assert_same_multiset(Chunk.concat(results, out_types), want)


def _case(lib, rng, W, jt, oir, sizes_b, sizes_p, nullable=True, sel_p=0.0, default=False, key_types=(INT64, INT64), key_pool=None,
          caps=None):
    btypes, ptypes = [key_types[0], INT64, INT64], [key_types[1], INT64, INT64]
    if key_pool is None:
        key_pool = rng.integers(-5000, 5000, 3000).astype(np.int64).view(np.uint64)
    bsh = _shards(rng, W, sizes_b, key_pool, 0, nullable, 0.1)
    psh = _shards(rng, W, sizes_p, np.concatenate([key_pool, key_pool + np.uint64(1 << 20)]), 10_000_000, nullable, 0.1)
    psel = [rng.random(n) >= sel_p for n in sizes_p] if sel_p else None
    di = [None, DEFAULT_ID, 7] if default and jt else None
    res = R.run(lib, W, jt, oir, btypes, ptypes, bsh, psh, psel, di, caps=caps)
    return res, (W, jt, oir, btypes, ptypes, bsh, psh, psel, di)


@pytest.mark.parametrize("W", [1, 2, 3, 8])
@pytest.mark.parametrize("jt,oir", JOINS)
def test_region_outer_join_matches_oracle(lib, W, jt, oir):
    """nullable keys and payloads on both sides, duplicate build keys, selected zeros, one empty shard and one whose keys
    are all NULL (W >= 2), then the same with defaultInner"""
    rng = np.random.default_rng(100 * W + 10 * jt + oir)
    sizes_b = [7_000 + 1_001 * s for s in range(W)]
    sizes_p = [20_000 + 3_001 * s for s in range(W)]
    if W >= 2:
        sizes_b[-1] = 0
        sizes_p[0] = 0
    res, args = _case(lib, rng, W, jt, oir, sizes_b, sizes_p, sel_p=0.1)
    _check(*args, res)
    res, args = _case(lib, rng, W, jt, oir, sizes_b, sizes_p, default=True)
    if W >= 2:                                   # a probe shard whose keys are all NULL
        args[6][1][1][0][:] = False
        res = R.run(lib, W, jt, oir, args[3], args[4], args[5], args[6], args[7], args[8])
    _check(*args, res)


@pytest.mark.parametrize("jt,oir", JOINS)
def test_region_outer_not_null_sides(lib, jt, oir):
    """no bitmaps at all: no mask word travels; an outer join still keeps its unselected rows local"""
    rng = np.random.default_rng(7 + jt)
    res, args = _case(lib, rng, 3, jt, oir, [9_000, 8_000, 7_000], [30_000, 0, 25_000], nullable=False, sel_p=0.2)
    _check(*args, res)


@pytest.mark.parametrize("jt,oir", JOINS)
def test_region_outer_signed_unsigned_and_float_zero(lib, jt, oir):
    """an INT64 probe key against a UINT64 build key with sign-bit values (equal bits, never equal values), and FLOAT64
    keys of +0.0 / -0.0 (two different keys)"""
    rng = np.random.default_rng(31 + jt)
    pool = np.concatenate([np.array([0, 1, 2, 1 << 63, (1 << 64) - 1, (1 << 63) + 5], np.uint64),
                           rng.integers(0, 1 << 62, 500).astype(np.uint64), rng.integers(1 << 63, (1 << 64) - 1, 500, dtype=np.uint64)])
    res, args = _case(lib, rng, 3, jt, oir, [3_000, 2_000, 1_000], [9_000, 8_000, 7_000], key_types=(UINT64, INT64), key_pool=pool)
    _check(*args, res)
    fpool = np.array([0.0, -0.0, 1.5, -2.25, np.inf, 1e300], np.float64).view(np.uint64)
    res, args = _case(lib, rng, 2, jt, oir, [500, 400], [4_000, 3_000], key_types=(FLOAT64, FLOAT64), key_pool=fpool)
    _check(*args, res)


@pytest.mark.parametrize("which", ["build", "probe", "miss"])
def test_region_cap_one_short_fails_the_gather(lib, which):
    """the exact-fit capacity minus one row, for the build regions, the probe regions or the kept miss rows: a gather that
    reads an overflowed slot (~0) fails with TQ_ERR_OOM and writes nothing (region_outer_ref checks the sentinels)"""
    rng = np.random.default_rng({"build": 1, "probe": 2, "miss": 3}[which])
    W = 3
    res, args = _case(lib, rng, W, 1, False, [6_000, 5_000, 4_000], [20_000, 15_000, 10_000], sel_p=0.1)
    _check(*args, res)
    _, jt, oir, btypes, ptypes, bsh, psh, psel, di = args
    bdest = [R.routed(c[0], n[0], None, W) for c, n in bsh]
    pdest = [R.routed(c[0], n[0], psel[s], W) for s, (c, n) in enumerate(psh)]
    bcap = max(int(np.sum(d == q)) for d in bdest for q in range(W))
    pcap = max(int(np.sum(d == q)) for d in pdest for q in range(W))
    mcap = max(int(np.sum(d < 0)) for d in pdest)
    caps = {"build": (bcap - 1, pcap, mcap), "probe": (bcap, pcap - 1, mcap), "miss": (bcap, pcap, mcap - 1)}[which]
    res = R.run(lib, W, jt, oir, btypes, ptypes, bsh, psh, psel, di, caps=caps)
    # an overflowing push publishes ~0 in every slot it writes (its own kept rows' slot and its regions on every rank), so
    # every destination has an overflowed slot to read
    assert all(r == L.TQ_ERR_OOM for r in res), res


def test_push_word_limit_refused_before_any_push(lib):
    """3 nullable columns (+ the mask word) or 4 NOT NULL columns fit the push's 4 words; 4 columns with one bitmap or 5
    NOT NULL columns are TQ_ERR_UNSUPPORTED_TYPE, and nothing lands in the regions or the slots"""
    rng = np.random.default_rng(5)
    n, W = 5_000, 2
    cols = [rng.integers(0, 1 << 40, n).astype(np.uint64) for _ in range(5)]
    nn = rng.random(n) >= 0.3
    keep = []
    try:
        for ncols, bm_col, ok in ((3, 2, True), (4, None, True), (4, 3, False), (5, None, False), (4, 0, False)):
            nns = [nn if c == bm_col else None for c in range(ncols)]
            src = R.Source(lib, cols[:ncols], nns)
            keep.append(src)
            nw = ncols + (bm_col is not None)
            reg = X.Regions(lib, W, nw, n)
            keep.append(reg)
            st = R.push(reg, 0, src, 0, 1)
            if st == L.TQ_OK:
                L.check(lib.tq_partition_push_sync(0))
            if ok:
                assert st == L.TQ_OK
                assert sum(reg.slots(d)[0][0] for d in range(W)) == int(np.sum(nns[0] if nns[0] is not None else np.ones(n, bool)))
            else:
                assert st == L.TQ_ERR_UNSUPPORTED_TYPE, (ncols, bm_col, st)
                assert all(reg.slots(d)[0] == (0, 0) for d in range(W)), "a refused push published a slot"
                assert all(np.all(reg.region(d, 0, c) == X.SENTINEL) for d in range(W) for c in range(reg.ncols[0])), "a refused push wrote rows"
    finally:
        for b in keep:
            b.free()
