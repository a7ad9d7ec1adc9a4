"""dist.BroadcastJoin with W ranks emulated in one process (TEST INFRASTRUCTURE): one sentinel-filled allocation holds the W
receive buffers of the broadcast's RegionLayout, and each emulated rank is a BroadcastJoin over a view of it that carries the
rank's number.  A step enqueues every rank's push (one push slot per rank), then joins rank by rank, as the ranks of
dist.BroadcastJoin.step_cols do across processes."""
import ctypes as C

import numpy as np

import exchange_ref as X
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, Chunk, Column, DeviceColumn
from tinysql_b200.dist import BroadcastJoin, RegionLayout


class EmuExchange(RegionLayout):
    """the W receive buffers of one broadcast table in one allocation; slots zeroed, regions at the sentinel"""

    def __init__(self, lib, world, table, pad_rows=0):
        super().__init__(lib, L, world, [table], pad_rows)
        self.buf = X.Buf(lib, world * self.bytes)
        self.bases = [self.buf.addr(d * self.bytes) for d in range(world)]
        for d in range(world):
            L.check(lib.tq_memset_device(C.c_void_p(self.slot_ptr(d, 0, 0)), 0, world * 16))
        X.compute_sync(lib)
        self.epoch = 0

    def next_epoch(self):
        self.epoch += 1
        return self.epoch

    def free(self):
        self.buf.free()


class RankView:
    """rank `rank`'s RegionExchange-like view of an EmuExchange"""

    def __init__(self, ex, rank):
        self.ex, self.rank = ex, rank

    def __getattr__(self, name):
        return getattr(self.ex, name)

    def wait(self, t):
        L.check(self.ex.lib.tq_region_wait(C.c_void_p(self.ex.slot_ptr(self.rank, t, 0)), self.ex.world, self.ex.epoch))


def shards(col, W, sizes=None):
    """col cut into W consecutive shards (sizes: rows per shard, default as even as possible)"""
    n = col.length
    if sizes is None:
        sizes = [n * (r + 1) // W - n * r // W for r in range(W)]
    bounds = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    assert bounds[-1] == n
    return [col.slice(int(bounds[r]), int(bounds[r + 1])) for r in range(W)]


def device(cols):
    return [DeviceColumn.from_host(c) for c in cols]


class Emulated:
    """W BroadcastJoins over one EmuExchange.  kw: the BroadcastJoin arguments after world / rank / n_build_max"""

    def __init__(self, lib, W, n_build_max, build_types, probe_types, **kw):
        self.lib, self.W = lib, W
        self.build_types, self.probe_types = list(build_types), list(probe_types)
        table = BroadcastJoin.table_of(self.build_types, n_build_max, kw.get("byte_caps") or [None] * len(self.build_types),
                                       int(bool(kw.get("build_nullable"))))
        self.ex = EmuExchange(lib, W, table)
        self.joins = [BroadcastJoin(lib, L, W, r, n_build_max, build_types, probe_types, slot=r, exchange=RankView(self.ex, r), **kw)
                      for r in range(W)]

    def step(self, bshards, pshards, psel=None):
        """bshards / pshards: per rank a list of host Columns.  Returns the per-rank result Chunks"""
        psel = psel or [None] * self.W
        keep = []
        try:
            self.ex.next_epoch()
            for r in range(self.W):
                b = device(bshards[r])
                keep += b
                self.joins[r].push(b)
            out = []
            for r in range(self.W):
                p = device(pshards[r])
                keep += p
                _, _, res = self.joins[r].join(p, selected=psel[r], keep_result=True)
                out.append(Chunk(res))
            return out
        finally:
            for r in range(self.W):
                L.check(self.lib.tq_partition_push_sync(r))
            for d in keep:
                d.free()

    def free(self):
        self.ex.free()


def concat(shard_lists, types):
    return Chunk.concat([Chunk(s) for s in shard_lists], types).cols


def nbytes(col):
    """cell bytes of a BYTES column (0 for the others)"""
    return sum(len(v) for v in col.values if v is not None) if col.tp == BYTES else 0


def byte_caps(types, bshards):
    """per build column, the most cell bytes one shard holds (None for 8-byte columns)"""
    return [max([nbytes(s[c]) for s in bshards] + [1]) if t == BYTES else None for c, t in enumerate(types)]


def empty_like(types):
    return [Column.empty(t, 0) for t in types]
