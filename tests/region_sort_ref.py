"""Reference side of the multi-GPU ORDER BY (tq_partition_push_sample / tq_partition_push_ranges / tq_sort_put_regions and
dist.RegionSort) — TEST INFRASTRUCTURE.

- The routing twin: a row's routing key is, per ByItem, the sort's key words (sort_ref.key_words) most significant first —
  the NULL flag, then the value word, or a string's 8-byte chunks first to last and then its length, each inverted when Desc
  — followed by the tie word (src_rank << 32) | row.  Its destination is the number of splitters whose key is at or below it.
- The sample positions' twin (range_sample_pos in csrc/scatter.cuh).
- Emulated: W RegionSorts over one allocation holding both tables (one push slot per rank), for the GPU suite."""
import ctypes as C

import numpy as np

import exchange_ref as X
import sort_ref as SR
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, Chunk, Column, DeviceColumn, DeviceVarColumn
from tinysql_b200.dist import RegionLayout, RegionSort

M64 = (1 << 64) - 1


def mix64(k):
    k &= M64
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & M64
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & M64
    k ^= k >> 33
    return k


def tie(src_rank, row):
    return (src_rank << 32) | row


def sample_pos(seed, src_rank, j, n, m):
    """row j of the sample of a shard of n rows (m = min(n, n_samples)): a hashed position inside stratum [j n / m, (j+1) n / m)"""
    lo, hi = j * n // m, (j + 1) * n // m
    return lo + mix64(seed ^ mix64(tie(src_rank, j))) % (hi - lo)


def routing_keys(by, vals, ties):
    """by: [(type, desc)] per ByItem; vals: per ByItem the Python values of the rows (None = NULL); ties: the rows' tie words.
    Returns one comparable tuple per row.  String chunks are padded to the longest string of `vals`, so keys built in one
    call compare as the sort's words do."""
    n = len(ties)
    parts = [[] for _ in range(n)]
    for (tp, desc), v in zip(by, vals):
        words = SR.key_words(tp, v, True)                 # [value] or [len, chunk 0 .., chunk k], then the NULL flag
        order = [words[-1]] + (words[1:-1] + [words[0]] if tp == BYTES else [words[0]])
        for i in range(n):
            parts[i] += [(M64 ^ w[i]) if desc else w[i] for w in order]
    return [tuple(p) + (t,) for p, t in zip(parts, ties)]


def range_dest(by, row_vals, row_ties, spl_vals, spl_ties):
    """the destination of every row: how many splitters have a routing key at or below the row's"""
    keys = routing_keys(by, [r + s for r, s in zip(row_vals, spl_vals)], list(row_ties) + list(spl_ties))
    rk, sk = keys[:len(row_ties)], keys[len(row_ties):]
    return [sum(1 for s in sk if s <= k) for k in rk]


def rows_of(cols):
    """host Columns -> list of row tuples of Python values (None = NULL)"""
    return Chunk(cols).rows()


def concat(shards, types):
    return Chunk.concat([Chunk(s) for s in shards], types).cols


def device(cols):
    return [DeviceVarColumn.from_host(c) if c.tp == BYTES else DeviceColumn.from_host(c) for c in cols]


class EmuTables(RegionLayout):
    """the W receive buffers of RegionSort's two tables in one allocation; slots zeroed, regions at the sentinel"""

    def __init__(self, lib, world, tables):
        super().__init__(lib, L, world, tables)
        self.buf = X.Buf(lib, world * self.bytes)
        self.bases = [self.buf.addr(d * self.bytes) for d in range(world)]
        for d in range(world):
            L.check(lib.tq_memset_device(C.c_void_p(self.slot_ptr(d, 0, 0)), 0, len(tables) * world * 16))
        X.compute_sync(lib)
        self.epoch = 0

    def next_epoch(self):
        self.epoch += 1
        return self.epoch

    def free(self):
        self.buf.free()


class RankView:
    """rank `rank`'s RegionExchange-like view of EmuTables"""

    def __init__(self, ex, rank):
        self.ex, self.rank = ex, rank

    def __getattr__(self, name):
        return getattr(self.ex, name)

    def wait(self, t):
        L.check(self.ex.lib.tq_region_wait(C.c_void_p(self.ex.slot_ptr(self.rank, t, 0)), self.ex.world, self.ex.epoch))


class Emulated:
    """W RegionSorts over one EmuTables (push slot r for rank r), driven phase by phase as W processes would run them"""

    def __init__(self, lib, W, types, by_cols, by_desc, n_max, byte_caps=None, nullable=True, limit_offset=0, limit_count=-1, n_samples=1024):
        self.lib, self.W, self.types = lib, W, list(types)
        tables = RegionSort.table_of(types, by_cols, n_max, byte_caps, nullable, n_samples)
        self.ex = EmuTables(lib, W, tables)
        self.sorts = [RegionSort(lib, L, W, r, types, by_cols, by_desc, n_max, byte_caps, nullable, limit_offset, limit_count, n_samples,
                                 slot=r, exchange=RankView(self.ex, r)) for r in range(W)]

    def step(self, shards):
        """shards: per rank a list of host Columns.  Returns per rank (rows, result host Columns); raises what the first
        failing rank raised, after every rank finished its part"""
        keep, out, err = [], [], None
        try:
            self.ex.next_epoch()
            dev = []
            for r in range(self.W):
                d = device(shards[r])
                keep += d
                dev.append(d)
            sort0 = self.sorts[0]
            if sort0.limit_count < 0:
                for r in range(self.W):
                    self.sorts[r].push_sample(dev[r])
            for r in range(self.W):
                self.sorts[r].push_rows(dev[r])
            for r in range(self.W):
                try:
                    out.append(self.sorts[r].finish(keep_result=True))
                except Exception as e:       # every rank runs its finish, as W processes would
                    err = err or e
                    out.append(None)
        finally:
            for s in self.sorts:
                s.release()
            for d in keep:
                d.free()
        if err is not None:
            raise err
        return out

    def free(self):
        self.ex.free()
