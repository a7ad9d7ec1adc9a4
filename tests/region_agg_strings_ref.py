"""Reference side of the string GROUP BY over the region exchange (tq_agg_push_partial_var / tq_agg_merge_regions_var), and
dist.RegionAgg with W ranks emulated in one process over broadcast_ref's EmuExchange (TEST INFRASTRUCTURE).

dest_of is the destination rule's twin for results that carry their GROUP BY items: a BYTES item contributes the string
dictionary's content hash of its bytes (dict_targets.sd_hash), NULL the NULL word, an 8-byte item its bits (region_agg_ref)."""
import numpy as np

import broadcast_ref as B
import dict_targets as D
import oracle_py as O
import region_agg_ref as RA
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, Chunk, DeviceColumn, DeviceVarColumn
from tinysql_b200.dist import RegionAgg, partial_var_cols

F64 = L.TQ_TYPE_FLOAT64


def item_words(col):
    """the 64-bit word each row of a GROUP BY item contributes (NULL rows are masked by the twin)"""
    if col.tp == BYTES:
        return D.sd_hashes(list(col.values))
    return np.ascontiguousarray(col.values).view(np.uint64)


def dest_of(key_cols, types, group_by, W):
    n = key_cols[0].length
    return RA.group_dest(n, [item_words(c) for c in key_cols], [c.not_null() for c in key_cols], [(types[g] & 0xFF) == F64 for g in group_by], W)


def rows_of(cols, skip=()):
    """the rows of host Columns as sorted tuples: NULL as None, REAL -0.0 as +0.0, a string as its bytes"""
    lists = []
    for i, c in enumerate(cols):
        if i in skip:
            continue
        vals = c.tolist() if c.tp == BYTES else [None if not ok else (float(v) + 0.0 if c.tp == F64 else int(v)) for v, ok in zip(c.values, c.not_null())]
        lists.append(vals)
    rows = list(zip(*lists)) if lists else []
    return sorted(rows, key=lambda r: tuple((x is None, repr(x)) for x in r))


def concat(shards, types):
    return Chunk.concat([Chunk(s) for s in shards], [t & 0xFF for t in types]).cols


def oracle(types, shards, group_by, funcs):
    rc, want = O.hash_agg([t & 0xFF for t in types], concat(shards, types), group_by, funcs)
    assert rc == 0, rc
    return want.cols


def byte_caps(types, group_by, funcs, shards):
    """per input column, the cell bytes of one rank's shard at most (the bound RegionAgg asks for), None for 8-byte columns"""
    srcs = {s for _, s in partial_var_cols(types, group_by, funcs)}
    return [max([sum(len(v) for v in sh[c].values) for sh in shards] + [1]) if c in srcs else None for c in range(len(types))]


def device(cols):
    return [DeviceVarColumn.from_host(c) if c.tp == BYTES else DeviceColumn.from_host(c) for c in cols]


class Emulated:
    """W RegionAggs over one EmuExchange (one push slot per rank)"""

    def __init__(self, lib, W, types, group_by, funcs, max_groups_per_rank, caps, ex=None):
        self.lib, self.W = lib, W
        w = RA.width(lib, RA.desc([t & 0xFF for t in types], group_by, funcs)[0])
        table, _ = RegionAgg.table_of(W, w, partial_var_cols(types, group_by, funcs), bool(group_by), max_groups_per_rank, caps)
        self.own = ex is None
        self.ex = ex or B.EmuExchange(lib, W, table)
        self.aggs = [RegionAgg(lib, L, W, r, types, group_by, funcs, max_groups_per_rank, slot=r, byte_caps=caps, exchange=B.RankView(self.ex, r))
                     for r in range(W)]

    def step(self, shards):
        """shards: per rank a list of host Columns.  Returns the per-rank results (host Columns, or None where a scalar
        aggregate is not finished)"""
        keep = []
        try:
            self.ex.next_epoch()
            for r in range(self.W):
                d = device(shards[r])
                keep += d
                self.aggs[r].push(d)
            return [self.aggs[r].finish(keep_result=True)[1] for r in range(self.W)]
        finally:
            for r in range(self.W):
                L.check(self.lib.tq_partition_push_sync(r))
            for d in keep:
                d.free()

    def free(self):
        if self.own:
            self.ex.free()
