"""Outer joins and nullable columns over the region exchange with W ranks emulated in one process (tests/exchange_ref.py's
Regions, on dist.RegionLayout): each source pushes its shards with tq_partition_push_regions, each destination copies its
regions with tq_region_gather and joins them with an ordinary join handle, as dist.RegionJoin does across processes; the
probe rows that cannot match stay on their source in a Regions of one rank, as RegionJoin keeps them.

A shard is (cols, nns): uint64 arrays and NOT-NULL bool arrays (None = no bitmap), key = column 0.  Every output buffer a
wrong count could reach is a sentinel-filled part of a larger allocation (GUARD rows before and after)."""
import ctypes as C

import numpy as np

import exchange_ref as X
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import Chunk, device_to_host
from tinysql_b200.dist import dest_rank_np

GUARD = 64


def routed(keys, nn, sel, n_parts):
    """destination of every row under the push's rule; -1 = cannot match (NULL key or selected == 0)"""
    d = dest_rank_np(np.asarray(keys).view(np.int64), n_parts) if len(keys) else np.zeros(0, np.int64)
    ok = np.ones(len(keys), bool)
    if nn is not None:
        ok &= nn
    if sel is not None:
        ok &= sel
    return np.where(ok, d, -1)


class GuardedCols:
    """ncols device columns of `rows` rows (+ bitmaps), each inside a sentinel-filled allocation"""

    def __init__(self, lib, ncols, rows, nullable):
        self.rows, self.ncols = rows, ncols
        self.bm_bytes = ((rows + 63) // 64) * 8
        self.data = [X.Buf(lib, (rows + 2 * GUARD) * 8) for _ in range(ncols)]
        self.bm = [X.Buf(lib, self.bm_bytes + 2 * GUARD) if nullable else None for _ in range(ncols)]
        self.arr = (L.TQColumn * ncols)()
        for c in range(ncols):
            self.arr[c].data = self.data[c].addr(GUARD * 8)
            self.arr[c].null_bitmap = self.bm[c].addr(GUARD) if self.bm[c] else None

    def guards_ok(self, n):
        """nothing written before the columns, past row n, or past the bitmap words of n rows"""
        for c in range(self.ncols):
            raw = self.data[c].get()
            if not (np.all(raw[:GUARD] == X.SENTINEL) and np.all(raw[GUARD + n:] == X.SENTINEL)):
                return False
            if self.bm[c] is not None:
                b = self.bm[c].get(np.uint8)
                used = ((n + 63) // 64) * 8
                if not (np.all(b[:GUARD] == X.SENTINEL_BYTE) and np.all(b[GUARD + used:] == X.SENTINEL_BYTE)):
                    return False
        return True

    def untouched(self):
        return all(np.all(b.get(np.uint8) == X.SENTINEL_BYTE) for b in self.data + [b for b in self.bm if b is not None])

    def read(self, n):
        """(values, not-null bools or None) per column"""
        out = []
        for c in range(self.ncols):
            v = self.data[c].get(np.uint64, GUARD * 8, n * 8)
            nn = None
            if self.bm[c] is not None:
                words = self.bm[c].get(np.uint8, GUARD, ((n + 63) // 64) * 8)
                nn = np.unpackbits(words, bitorder="little").astype(bool)
            out.append((v, nn))
        return out

    def free(self):
        for b in self.data + [b for b in self.bm if b is not None]:
            b.free()


class Source:
    """one emulated rank's shard in device memory: column pointers, bitmap pointers (padded to 64-row groups; None = no
    bitmap), selected bytes"""

    def __init__(self, lib, cols, nns, sel=None):
        self.n = len(cols[0])
        self.bufs, self.ptrs, self.bms = [], [], []
        for v, nn in zip(cols, nns):
            b = X.Buf(lib, max(self.n, 1) * 8, None)
            b.put(np.asarray(v).view(np.uint64))
            self.bufs.append(b)
            self.ptrs.append(b.addr())
            self.bms.append(None)
            if nn is not None:
                m = X.Buf(lib, ((self.n + 63) // 64) * 8 + 8, None)
                m.put(X.bitmap_words(nn))
                self.bufs.append(m)
                self.bms[-1] = m.addr()
        self.sel = None
        if sel is not None:
            s = X.Buf(lib, max(self.n, 1), None)
            s.put(np.asarray(sel, np.uint8))
            self.bufs.append(s)
            self.sel = s.addr()

    def free(self):
        for b in self.bufs:
            b.free()


def push(reg, src_idx, source, slot, epoch, miss=None):
    """source src_idx pushes its rows into its region on every destination of `reg` (wire columns = reg.ncols[0]); miss:
    (Regions of one rank, miss cap) keeps the rows that cannot match"""
    return reg.push(src_idx, source.ptrs, source.n, slot, epoch, bitmaps=source.bms, selected=source.sel, miss=miss)


def gather(lib, n_regions, slots_ptr, cap, ncols, has_mask, regs, out, out_cap=None):
    """tq_region_gather of the tq_column table regs ([region][wire column], RegionLayout.region_table) into GuardedCols
    `out`: (status, rows)"""
    n = C.c_int64(-1)
    st = lib.tq_region_gather(n_regions, C.c_void_p(slots_ptr), cap, ncols, has_mask, regs, out.arr, out.rows if out_cap is None else out_cap, C.byref(n))
    return st, n.value


def join_desc(jt, oir, btypes, ptypes, default_inner):
    tb = (C.c_int32 * len(btypes))(*btypes)
    tp = (C.c_int32 * len(ptypes))(*ptypes)
    k = (C.c_int32 * 1)(0)
    dbits = dnn = None
    if default_inner is not None:
        dt = {L.TQ_TYPE_INT64: np.int64, L.TQ_TYPE_UINT64: np.uint64, L.TQ_TYPE_FLOAT64: np.float64}
        dbits = (C.c_uint64 * len(btypes))(*[0 if v is None else int(np.array([v], dtype=dt[t]).view(np.uint64)[0]) for v, t in zip(default_inner, btypes)])
        dnn = (C.c_uint8 * len(btypes))(*[0 if v is None else 1 for v in default_inner])
    d = L.TQJoinDesc(jt, 1 if oir else 0, len(btypes), tb, len(ptypes), tp, 1, k, k, 0, 0,
                     C.cast(dbits, C.POINTER(C.c_uint64)) if dbits is not None else None, C.cast(dnn, C.POINTER(C.c_uint8)) if dnn is not None else None)
    return d, (tb, tp, k, dbits, dnn)


def local_join(lib, jt, oir, btypes, ptypes, default_inner, build, probes):
    """one destination's join: build = (GuardedCols, rows); probes = [(GuardedCols, rows, host selected or None)]"""
    d, keep = join_desc(jt, oir, btypes, ptypes, default_inner)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    out_types = (list(btypes) + list(ptypes)) if oir else (list(ptypes) + list(btypes))
    chunks = []
    try:
        if build[1]:
            L.check(lib.tq_join_put_build(h, build[0].arr, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        out = (L.TQColumn * len(out_types))()
        n, eof = C.c_int64(0), C.c_int32(0)
        for cols, rows, sel in probes:
            if not rows:
                continue
            s = None if sel is None else np.ascontiguousarray(sel, np.uint8)
            L.check(lib.tq_join_put_probe(h, cols.arr, None if s is None else s.ctypes.data, L.TQ_MEM_DEVICE))
            while True:                              # drain: the put borrows its columns until its batch is finished
                L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
                if n.value == 0:
                    break
                chunks.append(Chunk([device_to_host(out_types[c], out[c].data, out[c].null_bitmap, n.value) for c in range(len(out_types))]))
        L.check(lib.tq_join_probe_eof(h))
        while True:
            L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
            if n.value == 0:
                break
            chunks.append(Chunk([device_to_host(out_types[c], out[c].data, out[c].null_bitmap, n.value) for c in range(len(out_types))]))
    finally:
        lib.tq_join_destroy(h)
    return Chunk.concat(chunks, out_types)


def run(lib, W, jt, oir, btypes, ptypes, bshards, pshards, psel=None, default_inner=None, caps=None, epoch=1):
    """the whole exchange + join.  bshards / pshards: per source (cols, nns); psel: per source bool array or None.
    Returns (per destination result Chunk, refusal status or None).  caps = (build cap, probe cap, miss cap) overrides the
    exact-fit capacities; a gather that fails returns its status for that destination instead of a Chunk."""
    outer = jt != 0
    psel = psel or [None] * W
    bmask = int(any(nn is not None for cols, nns in bshards for nn in nns))
    pmask = int(any(nn is not None for cols, nns in pshards for nn in nns))
    nb, npc = len(btypes), len(ptypes)
    bdest = [routed(cols[0], nns[0], None, W) for cols, nns in bshards]
    pdest = [routed(cols[0], nns[0], psel[s], W) for s, (cols, nns) in enumerate(pshards)]
    cnt = lambda ds: max([int(np.sum(d == q)) for d in ds for q in range(W)] + [1])
    bcap, pcap, mcap = caps or (cnt(bdest), cnt(pdest), max([int(np.sum(d < 0)) for d in pdest] + [0]))
    breg, preg = X.Regions(lib, W, nb + bmask, bcap), X.Regions(lib, W, npc + pmask, pcap)
    nwp = npc + pmask
    keep, results = [], []
    try:
        srcs = [Source(lib, cols, nns) for cols, nns in bshards] + [Source(lib, cols, nns, psel[s]) for s, (cols, nns) in enumerate(pshards)]
        keep += srcs
        miss = [X.Regions(lib, 1, nwp, max(mcap, 1), GUARD) for _ in range(W)] if outer else []
        keep += miss
        for s in range(W):
            L.check(push(breg, s, srcs[s], s, epoch))
            L.check(push(preg, s, srcs[W + s], 8 + s, epoch, (miss[s], mcap) if outer else None))
        for slot in list(range(W)) + list(range(8, 8 + W)):
            L.check(lib.tq_partition_push_sync(slot))
        for d in range(W):
            L.check(breg.wait(d, epoch))
            L.check(preg.wait(d, epoch))
            gb = GuardedCols(lib, nb, W * bcap, bmask)
            gp = GuardedCols(lib, npc, W * pcap, pmask)
            gm = GuardedCols(lib, npc, max(mcap, 1), pmask)
            keep += [gb, gp, gm]
            st_b, rb = gather(lib, W, breg.slot_ptr(d, 0, 0), bcap, nb, bmask, breg.region_table(d, 0), gb)
            st_p, rp = gather(lib, W, preg.slot_ptr(d, 0, 0), pcap, npc, pmask, preg.region_table(d, 0), gp)
            st_m, rm = L.TQ_OK, 0
            if outer:
                L.check(miss[d].wait(0, epoch))
                st_m, rm = gather(lib, 1, miss[d].slot_ptr(0, 0, 0), max(mcap, 1), npc, pmask, miss[d].region_table(0, 0), gm)
            bad = [s for s in (st_b, st_p, st_m) if s != L.TQ_OK]
            if bad:
                for g, st, r in ((gb, st_b, rb), (gp, st_p, rp), (gm, st_m, rm)):
                    if st != L.TQ_OK:
                        assert g.untouched(), "a failed gather wrote into its outputs"
                results.append(bad[0])
                continue
            assert gb.guards_ok(rb) and gp.guards_ok(rp) and gm.guards_ok(rm), f"destination {d}: a gather wrote past its rows"
            probes = [(gp, rp, None)] + ([(gm, rm, np.zeros(rm, np.uint8))] if outer else [])
            results.append(local_join(lib, jt, oir, btypes, ptypes, default_inner, (gb, rb), probes))
        X.compute_sync(lib)
    finally:
        for b in keep:
            b.free()
        breg.free()
        preg.free()
    return results
