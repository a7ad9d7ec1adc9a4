"""Reference of the multi-GPU exchange, and the layout that runs it with every rank emulated in one process.

tq_partition_device: a row goes to dest_rank_np(key) (= (mix64(key) >> 40) % n_parts, dist.py), a row whose key is NULL to
row % n_parts; the rows of a partition keep their input order (a stable argsort by destination), so data, NOT-NULL bitmaps
and part_offsets compare bit for bit.

tq_partition_push_regions: a row whose key is NULL is neither counted nor sent; a destination receives a multiset of rows
(runs of a destination are claimed with atomics: the order inside it is not promised).

Regions: dist.RegionLayout of one table with all W ranks' receive buffers in one tq_device_alloc of W x layout.bytes
(rank d's at offset d x bytes), each region followed by `guard` rows of a sentinel (pad_rows), so a row written past the
cap lands inside the allocation and shows up in the guard instead of faulting."""
import ctypes as C

import numpy as np

from tinysql_b200 import _lib as L
from tinysql_b200.dist import RegionLayout, dest_rank_np

SENTINEL_BYTE = 0xA7
SENTINEL = np.uint64(0xA7A7A7A7A7A7A7A7)
EMPTY_KEY = np.uint64(0xA5C3F00DDEADBEEF)       # the join table's empty-slot marker: an ordinary key to the exchange
EDGE_KEYS = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1, EMPTY_KEY.view(np.int64),
                      np.float64(-0.0).view(np.int64), np.float64(0.0).view(np.int64), 1], dtype=np.int64)


# ------------------------------------------------------------------------------------------------ references
def partition_dest(keys, key_nn, n_parts):
    """destination of every row under tq_partition_device's rule"""
    n = len(keys)
    d = dest_rank_np(keys, n_parts) if n else np.zeros(0, np.int64)
    if key_nn is not None:
        rows = np.arange(n, dtype=np.int64)
        d = np.where(key_nn, d, rows % n_parts)
    return d


def partition_ref(cols, nns, key_col, n_parts):
    """cols: uint64 arrays; nns: NOT-NULL bool arrays or None.  Returns (out cols, out nns, part_offsets)."""
    d = partition_dest(cols[key_col].view(np.int64), nns[key_col], n_parts)
    order = np.argsort(d, kind="stable")
    offs = np.zeros(n_parts + 1, np.int64)
    offs[1:] = np.cumsum(np.bincount(d, minlength=n_parts))
    return [c[order] for c in cols], [None if m is None else m[order] for m in nns], offs


def push_dest(keys, key_nn, n_parts):
    """destination of every row under the push rule; -1 = not sent (NULL key)"""
    d = dest_rank_np(keys, n_parts) if len(keys) else np.zeros(0, np.int64)
    if key_nn is not None:
        d = np.where(key_nn, d, -1)
    return d


def rows_of(cols, idx):
    """the rows idx of cols as one (len(idx), ncols) uint64 matrix, sorted (a multiset in canonical order)"""
    m = np.stack([np.asarray(c).view(np.uint64)[idx] for c in cols], axis=1) if len(cols) else np.zeros((len(idx), 0), np.uint64)
    return m[np.lexsort(m.T[::-1])] if len(m) else m


def sorted_rows(m):
    return m[np.lexsort(m.T[::-1])] if len(m) else m


def keys_to(rng, n_parts, target, n, pool=1 << 18):
    """n distinct int64 keys whose destination (dest_rank_np) is `target`"""
    out = []
    while sum(len(x) for x in out) < n:
        k = rng.integers(-(1 << 63), (1 << 63) - 1, pool, dtype=np.int64)
        out.append(k[dest_rank_np(k, n_parts) == target])
    k = np.unique(np.concatenate(out))
    return rng.permutation(k)[:n]


# ------------------------------------------------------------------------------------------------ device memory
def compute_sync(lib):
    """wait for the library's compute stream (tq_memset_device is queued there); the emulation runs everything inline"""
    try:
        fn = lib.tq_compute_synchronize
    except AttributeError:
        return
    L.check(fn())


class Buf:
    """one tq_device_alloc of `nbytes`, prefilled with the sentinel byte"""

    def __init__(self, lib, nbytes, fill=SENTINEL_BYTE):
        self.lib, self.nbytes = lib, int(nbytes)
        self.p = C.c_void_p()
        L.check(lib.tq_device_alloc(max(self.nbytes, 8), C.byref(self.p)))
        if fill is not None:
            L.check(lib.tq_memset_device(self.p, fill, max(self.nbytes, 8)))
        compute_sync(lib)

    def addr(self, byte_off=0):
        return self.p.value + int(byte_off)

    def put(self, a, byte_off=0):
        a = np.ascontiguousarray(a)
        if a.nbytes:
            L.check(self.lib.tq_memcpy_h2d(C.c_void_p(self.addr(byte_off)), a.ctypes.data, a.nbytes))

    def get(self, dtype=np.uint64, byte_off=0, nbytes=None):
        nbytes = self.nbytes - byte_off if nbytes is None else int(nbytes)
        out = np.empty(nbytes // np.dtype(dtype).itemsize, dtype)
        if out.nbytes:
            L.check(self.lib.tq_memcpy_d2h(out.ctypes.data, C.c_void_p(self.addr(byte_off)), out.nbytes))
        return out

    def free(self):
        if self.p:
            self.lib.tq_device_free(self.p)
            self.p = C.c_void_p()


def bitmap_words(nn):
    """NOT-NULL bools -> the device bitmap (bit r of 32-bit word r >> 5), as bytes padded to whole 8-byte words"""
    b = np.packbits(np.asarray(nn, bool), bitorder="little")
    pad = ((len(nn) + 63) // 64) * 8
    return np.concatenate([b, np.zeros(pad - len(b), np.uint8)])


class Regions(RegionLayout):
    """W emulated ranks' receive buffers of one table (t = 0): slots start at zero (epoch 0: nothing published), regions and
    guards at the sentinel.  words: words per wire column when they are not cap each (dist.RegionAgg.table_of's var-len
    layout)."""

    def __init__(self, lib, world, ncols, cap, guard=64, words=None):
        super().__init__(lib, L, world, [(ncols, cap) if words is None else (ncols, cap, words)], pad_rows=guard)
        self.buf = Buf(lib, world * self.bytes)
        self.bases = [self.buf.addr(d * self.bytes) for d in range(world)]
        for d in range(world):
            L.check(lib.tq_memset_device(C.c_void_p(self.slot_ptr(d, 0, 0)), 0, world * 16))
        compute_sync(lib)

    def push(self, src, cols, n, slot, epoch, key_col=0, bitmaps=None, selected=None, miss=None):
        """source `src` scatters its n rows (device column pointers; bitmaps: a device NULL bitmap pointer or None per
        column) into its region on every destination.  selected: device bytes or None.  miss: (Regions of one rank, miss
        cap) that keeps the rows which cannot match on the source (keep_misses); without it they are dropped."""
        dest, cnts = self.push_tables(0, src)
        tq = (L.TQColumn * len(cols))()
        for c in range(len(cols)):
            tq[c].length, tq[c].data = n, cols[c]
            tq[c].null_bitmap = bitmaps[c] if bitmaps else None
        md, ms, mcap = (None, None, 0) if miss is None else (miss[0].push_tables(0, 0)[0], miss[0].slot_ptr(0, 0, 0), miss[1])
        return self.lib.tq_partition_push_regions(len(cols), tq, key_col, n, self.world, selected, int(miss is not None), dest, cnts, self.cap[0],
                                                  md, ms, mcap, slot, epoch)

    def wait(self, dst, epoch):
        return self.lib.tq_region_wait(C.c_void_p(self.slot_ptr(dst, 0, 0)), self.world, epoch)

    def slots(self, dst):
        """[(rows, epoch)] of every source on `dst` (host read)"""
        return [(int(r), int(e)) for r, e in self.read_slots(dst)[0]]

    def region(self, dst, src, c):
        """the region's words (cap rows, unless the layout lists its own) followed by its guard rows"""
        offs = self.col_off[0] + [self.stride[0]]
        out = np.empty(offs[c + 1] - offs[c], np.uint64)
        L.check(self.lib.tq_memcpy_d2h(out.ctypes.data, C.c_void_p(self.region_ptr(dst, 0, src, c)), out.nbytes))
        return out

    def free(self):
        self.buf.free()
