"""Reference of the GROUP BY over the region exchange (tq_agg_push_partial / tq_agg_merge_regions), and the runner that drives
it with every rank emulated in one process on exchange_ref's Regions, whose argument tables are dist.RegionLayout's.

group_dest is the Python twin of the destination rule (include/tinysql_b200.h, csrc/scatter.cuh): h = 0, then per GROUP BY
item h = mix64(h ^ v), v = the item's 8 bytes (REAL: -0.0 read as +0.0) or GROUP_NULL_WORD for NULL; rank = (h >> 40) % W."""
import ctypes as C
from collections import namedtuple

import numpy as np

import exchange_ref as X
import int_agg_ref as I
import oracle_py as O
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, Chunk, Column
from tinysql_b200.dist import _tq_device, agg_drain, mix64_np, partial_var_cols

GROUP_NULL_WORD = np.uint64(0x4E554C4C4E554C4C)
NEG_ZERO = np.uint64(1 << 63)
NP_TYPE = {L.TQ_TYPE_INT64: np.int64, L.TQ_TYPE_UINT64: np.uint64, L.TQ_TYPE_FLOAT64: np.float64}


def group_dest(n, items, nns, reals, n_parts):
    """destination of n partial rows; items: the GROUP BY columns as uint64 arrays, nns: NOT-NULL bool arrays or None,
    reals: per item, whether it is REAL"""
    h = np.zeros(n, np.uint64)
    for v, nn, real in zip(items, nns, reals):
        v = np.asarray(v).view(np.uint64)
        if real:
            v = np.where(v == NEG_ZERO, np.uint64(0), v)
        if nn is not None:
            v = np.where(nn, v, GROUP_NULL_WORD)
        h = mix64_np(h ^ v)
    return ((h >> np.uint64(40)) % np.uint64(n_parts)).astype(np.int64)


# ------------------------------------------------------------------------------------------------ emulated ranks
def desc(types, group_by, funcs, not_null=()):
    """a tq_agg_desc (and what keeps its arrays alive); not_null: input columns declared NOT NULL"""
    it = (C.c_int32 * len(types))(*[t | (L.TQ_TYPE_NOT_NULL if c in not_null else 0) for c, t in enumerate(types)])
    gb = (C.c_int32 * max(len(group_by), 1))(*group_by)
    fa = (L.TQAggFunc * max(len(funcs), 1))(*[L.TQAggFunc(f, a) for f, a in funcs])
    return L.TQAggDesc(len(types), it, len(group_by), gb, len(funcs), fa, 0), (it, gb, fa)


def create(lib, d):
    h = C.c_void_p()
    L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
    return h


def width(lib, d):
    h = create(lib, d)
    try:
        w = C.c_int32(0)
        L.check(lib.tq_agg_partial_width(h, C.byref(w)))
        return w.value
    finally:
        lib.tq_agg_destroy(h)


def partial_handle(lib, d, src):
    """a Partial1 handle fed one shard (an R.Source in device memory, or a list of DeviceColumn / DeviceVarColumn), eof'd"""
    h = create(lib, d)
    if not hasattr(src, "ptrs"):
        arr, n = _tq_device(L, src)
        if n:
            L.check(lib.tq_agg_put(h, arr, L.TQ_MEM_DEVICE))
    elif src.n:
        arr = (L.TQColumn * len(src.ptrs))()
        for c in range(len(src.ptrs)):
            arr[c].length, arr[c].data, arr[c].null_bitmap = src.n, src.ptrs[c], src.bms[c]
        L.check(lib.tq_agg_put(h, arr, L.TQ_MEM_DEVICE))
    L.check(lib.tq_agg_eof(h))
    return h


def var_region_table(reg, dst, w, var_cols):
    """destination dst's regions as tq_agg_merge_regions_var takes them (dist.RegionAgg.merge_table): a var-len column c has
    .offsets = its word area and .data = its byte area (wire area w + 1 + v)"""
    regs = reg.region_table(dst, 0)
    nw, nc = w + 1, reg.ncols[0]
    out = (L.TQColumn * (reg.world * nw))()
    for g in range(reg.world):
        for c in range(nw):
            out[g * nw + c].length, out[g * nw + c].data = reg.cap[0], regs[g * nc + c].data
        for v, (c, _) in enumerate(var_cols):
            out[g * nw + c].offsets = out[g * nw + c].data
            out[g * nw + c].data = regs[g * nc + nw + v].data
    return out


def run(lib, W, types, group_by, funcs, shards, reg, epoch=1, not_null=(), statuses=False, byte_cap=None):
    """one step: every source's Partial1 handle pushes (slot = source), every destination waits and merges into a Final handle.
    shards: per source an R.Source (or a list of device columns).  Returns per destination (status of tq_agg_merge_regions,
    host Columns or None).  A scalar aggregate is finished on destination 0 only (dist.RegionAgg): the others return None.
    statuses: nothing raises on a failed push or drain; returns (the push status of every source, per destination (merge
    status, status of tq_agg_next_device / tq_agg_next, host Columns or None)).  byte_cap: run the _var pair with these
    byte caps on a reg laid out as dist.RegionAgg.table_of."""
    d, keep = desc(types, group_by, funcs, not_null)
    var = byte_cap is not None
    if var:
        w, var_cols = width(lib, d), partial_var_cols(types, group_by, funcs)
        caps = (C.c_int64 * max(len(byte_cap), 1))(*byte_cap)
    hs, pushed = [], []
    try:
        for s in range(W):
            hs.append(partial_handle(lib, d, shards[s]))
            dest, cnts = reg.push_tables(0, s)
            if var:
                st = lib.tq_agg_push_partial_var(hs[-1], W, dest, cnts, reg.cap[0], caps, s, epoch)
            else:
                st = lib.tq_agg_push_partial(hs[-1], W, dest, cnts, reg.cap[0], s, epoch)
            if not statuses:
                L.check(st)
            pushed.append(st)
        out = []
        for q in range(W):
            L.check(reg.wait(q, epoch))                      # queued after every push that satisfies it
            hf = create(lib, d)
            try:
                slots = C.c_void_p(reg.slot_ptr(q, 0, 0))
                if var:
                    st = lib.tq_agg_merge_regions_var(hf, W, slots, reg.cap[0], var_region_table(reg, q, w, var_cols))
                else:
                    st = lib.tq_agg_merge_regions(hf, W, slots, reg.cap[0], reg.region_table(q, 0))
                if st != L.TQ_OK:
                    out.append((st, None, None) if statuses else (st, None))
                    continue
                L.check(lib.tq_agg_eof(hf))
                if not statuses:
                    out.append((st, agg_drain(lib, L, hf, len(funcs)) if group_by or q == 0 else None))
                    continue
                nxt, cols = L.TQ_OK, None
                if group_by or q == 0:
                    try:
                        cols = agg_drain(lib, L, hf, len(funcs))
                    except L.TQError as e:
                        nxt = e.status
                out.append((st, nxt, cols))
            finally:
                lib.tq_agg_destroy(hf)
        for s in range(W):
            L.check(lib.tq_partition_push_sync(s))
    finally:
        for h in hs:
            lib.tq_agg_destroy(h)
    return (pushed, out) if statuses else out


# ------------------------------------------------------------------------------------------------ comparison
def canon(cols, skip=()):
    """rows of host Columns as one uint64 matrix (NULL = 0 with a 0 flag column, REAL -0.0 as +0.0), rows sorted; columns in
    skip are left out"""
    m = []
    for i, c in enumerate(cols):
        if i in skip:
            continue
        nn = c.not_null()
        v = np.asarray(c.values)
        if v.dtype == np.float64:
            v = v + 0.0
        bits = np.where(nn, np.ascontiguousarray(v).view(np.uint64), np.uint64(0))
        m += [nn.astype(np.uint64), bits]
    if not m:
        return np.zeros((cols[0].length if cols else 0, 0), np.uint64)
    return X.sorted_rows(np.stack(m, axis=1))


def oracle(types, shards_host, group_by, funcs):
    """O.hash_agg over the concatenation of every shard: shards_host = per source (value arrays, NOT-NULL arrays or None)"""
    cols = []
    for c, t in enumerate(types):
        vals = np.concatenate([np.asarray(v[c]).view(NP_TYPE[t]) for v, _ in shards_host]) if shards_host else np.zeros(0, NP_TYPE[t])
        nns = [nn[c] if nn[c] is not None else np.ones(len(v[c]), bool) for v, nn in shards_host]
        cols.append(Column(t, vals, np.concatenate(nns) if nns else np.zeros(0, bool)))
    rc, want = O.hash_agg(types, cols, group_by, funcs)
    assert rc == 0, rc
    return want


# ------------------------------------------------------------------------------------------------ expectations per rank
def key_dest(labels, key_types, W):
    """the rank the destination twin names for each group key tuple of int_agg_ref.expect (None = NULL, bytes for a BYTES
    item: its dictionary content hash); rank 0 for a scalar aggregate"""
    import dict_targets as D
    n = len(labels)
    if not key_types:
        return np.zeros(n, np.int64)
    items, nns = [], []
    for i, t in enumerate(key_types):
        vals = [lab[i] for lab in labels]
        nns.append(np.array([v is not None for v in vals], bool))
        if (t & 0xFF) == BYTES:
            items.append(D.sd_hashes([b"" if v is None else v for v in vals]))
        elif (t & 0xFF) == L.TQ_TYPE_FLOAT64:
            items.append(np.array([0.0 if v is None else v for v in vals], np.float64).view(np.uint64))
        else:
            items.append(np.array([0 if v is None else v % (1 << 64) for v in vals], dtype=object).astype(np.uint64))
    return group_dest(n, items, nns, [(t & 0xFF) == L.TQ_TYPE_FLOAT64 for t in key_types], W)


RankExpect = namedtuple("RankExpect", "push_fail dest_fail ranks")
"""push_fail: the sources whose push must fail (a partial total of theirs leaves int64: int_agg_ref.expect_partial raises),
and then every destination's merge fails; dest_fail (no push failing): the ranks that finish a group whose merged total
leaves int64, whose next fails; ranks[q]: int_agg_ref.Expected of the groups rank q finishes"""


def expect_ranks(types, rank_cols, group_by, funcs, W):
    """where every failure of one step lands, and the exact groups of every other rank.  rank_cols: per source its input
    Columns (BIGINT / BIGINT UNSIGNED arguments, keys of any type)"""
    push_fail = set()
    for r, cols in enumerate(rank_cols):
        if cols[0].length:
            try:
                I.expect_partial(types, cols, group_by, funcs)
            except OverflowError:
                push_fail.add(r)
    full = Chunk.concat([Chunk(c) for c in rank_cols], types).cols
    want = I.expect(full, group_by, funcs)
    labels = list(want.groups)
    d = key_dest(labels, [types[g] for g in group_by], W)
    owner = dict(zip(labels, d.tolist()))
    dest_fail = set() if push_fail else {owner[k] for k in want.over}
    ranks = [I.Expected({k: v for k, v in want.groups.items() if owner[k] == q}, False) for q in range(W)]
    return RankExpect(push_fail, dest_fail, ranks)
