"""The multi-GPU exchange on one GPU, every rank emulated in this process with its receive buffers in local HBM, against the
exact reference of tests/exchange_ref.py:

  A. tq_partition_device (the NCCL path's and the distributed GROUP BY's partitioner): stable, NULL keys to row % n_parts,
     bitmaps carried with their rows, bit for bit at the warp-chunk (2048 rows) and block (16384 rows) edges, 1..256
     partitions and 1..16 columns; nothing written outside the outputs; FLOAT32 / BYTES columns refused.
  B. tq_partition_push_regions -> the published {rows, epoch} slots -> tq_region_wait: every destination's rows exact with
     the guard rows after them intact, at 0..1,100,003 rows, 1..8 destinations and 1..4 columns; NULL keys neither counted
     nor sent; 1..8 emulated ranks with caps that fit, fit exactly and overflow by one row; two pushes queued on one slot
     behind a busy push stream each keep their own regions and slots; every bad argument refused before anything is written.
  C. tq_join_put_probe_segments over regions filled by real pushes, in the exchange's order (push, device-side wait, join).
  D. dist.py's device GROUP BY and join with the NCCL exchange replaced by concatenating each destination's slices.

Every buffer a wrong offset or cap could reach is a sentinel-filled part of a larger allocation, so such a bug misplaces
rows inside an allocation and shows up in a guard.  Every tq_region_wait is queued after the pushes that satisfy it.
Section A's bodies also run under the CPU emulation (tests/test_emu_exchange.py)."""
import ctypes as C

import numpy as np
import pytest

import exchange_ref as X
import oracle_py as O
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import FLOAT64, INT64, Column
from tinysql_b200.dist import dest_rank_np
from util import assert_same_multiset

pytestmark = pytest.mark.gpu

GUARD = 64                     # sentinel rows around every output
PART_TYPES = (L.TQ_TYPE_INT64, L.TQ_TYPE_UINT64 | L.TQ_TYPE_NOT_NULL, L.TQ_TYPE_FLOAT64)


# ================================================================================================ A. tq_partition_device
class _PartIO:
    """inputs and sentinel-guarded outputs of one tq_partition_device call"""

    def __init__(self, lib, cols, nns):
        self.lib, self.n, self.ncols, self.cols, self.nns = lib, len(cols[0]), len(cols), cols, nns
        n = self.n
        self.bm_bytes = ((n + 63) // 64) * 8          # what the kernel may touch of an output bitmap
        self.bufs, self.inp, self.out = [], (L.TQColumn * self.ncols)(), (L.TQColumn * self.ncols)()
        self.out_data, self.out_bm = [], []
        for c in range(self.ncols):
            d = self._buf(n * 8, None)
            d.put(cols[c])
            self.inp[c].length, self.inp[c].data = n, d.addr()
            if nns[c] is not None:
                b = self._buf(self.bm_bytes + 8, None)
                b.put(X.bitmap_words(nns[c]))
                self.inp[c].null_bitmap = b.addr()
            od = self._buf((n + 2 * GUARD) * 8)
            self.out[c].data = od.addr(GUARD * 8)
            self.out_data.append(od)
            ob = None
            if nns[c] is not None:
                ob = self._buf(self.bm_bytes + 2 * GUARD)
                self.out[c].null_bitmap = ob.addr(GUARD)
            self.out_bm.append(ob)

    def _buf(self, nbytes, fill=X.SENTINEL_BYTE):
        b = X.Buf(self.lib, nbytes, fill)
        self.bufs.append(b)
        return b

    def run(self, types, key_col, n_parts, n=None):
        self.offs = (C.c_int64 * (n_parts + 1))(*([-7] * (n_parts + 1)))
        t = (C.c_int32 * self.ncols)(*types)
        return self.lib.tq_partition_device(self.ncols, self.inp, t, key_col, self.n if n is None else n, n_parts, self.out, self.offs)

    def result(self):
        """(out data, out bitmap bytes, guards intact?) per column"""
        n, res = self.n, []
        for c in range(self.ncols):
            raw = self.out_data[c].get()
            data_ok = np.all(raw[:GUARD] == X.SENTINEL) and np.all(raw[GUARD + n:] == X.SENTINEL)
            bm = None
            if self.out_bm[c] is not None:
                rb = self.out_bm[c].get(np.uint8)
                data_ok = data_ok and np.all(rb[:GUARD] == X.SENTINEL_BYTE) and np.all(rb[GUARD + self.bm_bytes:] == X.SENTINEL_BYTE)
                bm = rb[GUARD:GUARD + self.bm_bytes]
            res.append((raw[GUARD:GUARD + n], bm, data_ok))
        return res

    def untouched(self):
        return all(np.all(b.get(np.uint8) == X.SENTINEL_BYTE) for b in self.out_data + [b for b in self.out_bm if b is not None])

    def free(self):
        for b in self.bufs:
            b.free()


def _gen_part_cols(rng, n, ncols, key_col, key_nullable, payload_nullable, keys=None):
    cols = [rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64).view(np.uint64) for _ in range(ncols)]
    if keys is not None:
        cols[key_col] = np.asarray(keys, np.int64).view(np.uint64)
    elif n:
        edge = rng.random(n) < 0.05
        cols[key_col][edge] = rng.choice(X.EDGE_KEYS, int(edge.sum())).view(np.uint64)
    nns = [None] * ncols
    for c in range(ncols):
        if (c == key_col and key_nullable) or (c != key_col and payload_nullable and c % 2 == 0):
            nns[c] = rng.random(n) >= (0.2 if c == key_col else 0.35)
    return cols, nns


def _check_partition(lib, rng, n, n_parts, ncols, key_col, key_nullable, payload_nullable, keys=None, io=None):
    own = io is None
    if own:
        io = _PartIO(lib, *_gen_part_cols(rng, n, ncols, key_col, key_nullable, payload_nullable, keys))
    cols, nns = io.cols, io.nns
    try:
        types = [PART_TYPES[c % 3] for c in range(ncols)]
        L.check(io.run(types, key_col, n_parts))
        want_cols, want_nns, want_offs = X.partition_ref(cols, nns, key_col, n_parts)
        assert list(io.offs) == list(want_offs), f"part_offsets n={n} n_parts={n_parts}"
        for c, (data, bm, guards_ok) in enumerate(io.result()):
            assert guards_ok, f"column {c}: a write outside the output (n={n}, n_parts={n_parts})"
            assert np.array_equal(data, want_cols[c]), f"column {c} data, n={n} n_parts={n_parts}"
            if want_nns[c] is not None:
                assert np.array_equal(bm, X.bitmap_words(want_nns[c])), f"column {c} bitmap (bits >= n must be 0), n={n} n_parts={n_parts}"
    finally:
        if own:
            io.free()


SIZES = [0, 1, 2047, 2048, 2049, 16383, 16384, 16385, 1_000_003]
PARTS = [1, 2, 3, 7, 8, 64, 255, 256]


@pytest.mark.parametrize("n", SIZES)
def test_partition_matches_stable_reference(lib, n):
    """every partition count at one size: 1, 2 or 16 columns with the key not in column 0 (when there are several), a
    nullable key on every other call and nullable payload columns, keys salted with the int64 / EMPTY_KEY / -0.0 edges"""
    rng = np.random.default_rng(n + 11)
    for i, n_parts in enumerate(PARTS):
        ncols = (1, 2, 16)[i % 3]
        key_col = ncols - 1 if i % 2 == 0 else ncols // 2
        _check_partition(lib, rng, n, n_parts, ncols, key_col, key_nullable=i % 2 == 0, payload_nullable=i % 4 < 2)


def test_partition_edge_keys_and_skew(lib, n=20000):
    """only edge keys (INT64_MIN / MAX, 0, -1, EMPTY_KEY, +-0.0 bits); then keys aimed so every row goes to one partition
    and the others stay empty, for the first, a middle and the last partition"""
    rng = np.random.default_rng(3)
    for n_parts in (2, 7, 256):
        _check_partition(lib, rng, n, n_parts, 3, 1, True, True, keys=rng.choice(X.EDGE_KEYS, n))
        for target in (0, n_parts // 2, n_parts - 1):
            aimed = X.keys_to(rng, n_parts, target, 512)
            _check_partition(lib, rng, n, n_parts, 2, 1, False, True, keys=rng.choice(aimed, n))
            _check_partition(lib, rng, n, n_parts, 2, 1, True, False, keys=rng.choice(aimed, n))


def test_partition_scratch_reuse(lib, big=40000, small=3001):
    """a large call, then a smaller one through the same static scratch (counts, scan): no stale count of the large call
    leaks into the small one"""
    rng = np.random.default_rng(4)
    _check_partition(lib, rng, big, 256, 2, 1, True, True)
    _check_partition(lib, rng, small, 256, 2, 1, True, True)
    _check_partition(lib, rng, small, 3, 2, 0, True, True)
    _check_partition(lib, rng, big, 5, 2, 1, False, False)


def test_partition_refusals(lib):
    """bad shapes: TQ_ERR_INVALID_ARG; a column the kernels cannot move as 8-byte words (FLOAT32, BYTES, offsets set):
    TQ_ERR_UNSUPPORTED_TYPE.  Either way nothing is written."""
    rng = np.random.default_rng(5)
    n = 1000
    cols, nns = _gen_part_cols(rng, n, 3, 1, True, True)
    io = _PartIO(lib, cols, nns)
    ok = [L.TQ_TYPE_INT64] * 3
    try:
        for n_parts in (0, 257, -1):
            assert io.run(ok, 1, n_parts) == L.TQ_ERR_INVALID_ARG
        for key_col in (-1, 3):
            assert io.run(ok, key_col, 4) == L.TQ_ERR_INVALID_ARG
        t0 = (C.c_int32 * 17)(*([L.TQ_TYPE_INT64] * 17))
        offs = (C.c_int64 * 5)()
        assert lib.tq_partition_device(0, io.inp, t0, 0, n, 4, io.out, offs) == L.TQ_ERR_INVALID_ARG
        wide_in, wide_out = (L.TQColumn * 17)(*([io.inp[0]] * 17)), (L.TQColumn * 17)(*([io.out[0]] * 17))
        assert lib.tq_partition_device(17, wide_in, t0, 0, n, 4, wide_out, offs) == L.TQ_ERR_INVALID_ARG
        saved = io.out[2].null_bitmap
        io.out[2].null_bitmap = None                                   # column 2 has an input bitmap
        assert io.run(ok, 1, 4) == L.TQ_ERR_INVALID_ARG
        io.out[2].null_bitmap = saved
        for bad in (L.TQ_TYPE_FLOAT32, L.TQ_TYPE_BYTES, L.TQ_TYPE_FLOAT32 | L.TQ_TYPE_NOT_NULL):
            for c in range(3):
                types = list(ok)
                types[c] = bad
                assert io.run(types, 1, 4) == L.TQ_ERR_UNSUPPORTED_TYPE, (bad, c)
        io.inp[0].offsets = io.inp[0].data                             # a var-len layout, whatever its declared type
        assert io.run(ok, 1, 4) == L.TQ_ERR_UNSUPPORTED_TYPE
        io.inp[0].offsets = None
        assert io.untouched(), "a refused call wrote into its outputs"
        assert list(io.offs) == [-7] * 5, "a refused call wrote part_offsets"
        _check_partition(lib, rng, n, 4, 3, 1, True, True, io=io)      # the same buffers still partition correctly
    finally:
        io.free()


# ================================================================================================ B. push_regions / publish / wait
def _dev_cols(lib, arrays, keep):
    ptrs = []
    for a in arrays:
        b = X.Buf(lib, max(len(a), 1) * 8, None)
        b.put(np.asarray(a).view(np.uint64))
        keep.append(b)
        ptrs.append(b.addr())
    return ptrs


def _tq(ptrs, n):
    arr = (L.TQColumn * len(ptrs))()
    for c, p in enumerate(ptrs):
        arr[c].length, arr[c].data = n, p
    return arr


def _push_data(rng, n, ncols, key_col, first_id):
    cols = [np.arange(first_id, first_id + n, dtype=np.int64) * (c + 3) + c for c in range(ncols)]
    k = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64)
    edge = rng.random(n) < 0.02
    k[edge] = rng.choice(X.EDGE_KEYS, int(edge.sum()))
    cols[key_col] = k
    return cols


def _check_source(reg, s, cols, dest, epoch):
    """source s's slot and region on every destination after a push that did not overflow: dest[i] = where row i went
    (-1 = not sent); each region holds exactly those rows (a multiset, whole rows) and the sentinel past them"""
    for d in range(reg.world):
        idx = np.flatnonzero(dest == d)
        assert reg.slots(d)[s] == (len(idx), epoch), f"slot ({d}, {s})"
        got = np.stack([reg.region(d, s, c) for c in range(reg.ncols[0])], axis=1)
        assert np.all(got[len(idx):] == X.SENTINEL), f"region ({d}, {s}): a row past its count"
        assert np.array_equal(X.sorted_rows(got[:len(idx)]), X.rows_of(cols, idx)), f"region ({d}, {s}) rows"


def _push_one_source(lib, cols, ptrs, key_col, n_parts, key_nn=None, key_bm=None):
    """one source pushes every row into n_parts destinations whose regions fit exactly; with key_bm (the device bitmap of
    key_nn) on the key column the mask word travels as the last wire column and says NOT NULL for every sent row"""
    n = len(cols[0])
    dest = X.push_dest(cols[key_col], key_nn, n_parts)
    cap = max(int(np.bincount(dest[dest >= 0], minlength=n_parts).max()) if n else 0, 1)
    mask = [] if key_bm is None else [np.full(n, (1 << len(cols)) - 1, np.uint64)]
    reg = X.Regions(lib, n_parts, len(cols) + len(mask), cap, guard=GUARD)
    try:
        bms = None if key_bm is None else [key_bm if c == key_col else None for c in range(len(cols))]
        L.check(reg.push(0, ptrs, n, 0, 5, key_col, bms))
        L.check(lib.tq_partition_push_sync(0))
        _check_source(reg, 0, cols + mask, dest, 5)
        assert all(reg.slots(d)[1:] == [(0, 0)] * (n_parts - 1) for d in range(n_parts)), "a slot of another source was written"
    finally:
        reg.free()


@pytest.mark.parametrize("n", [0, 1, 4095, 4096, 4097, 1_100_003])
def test_push_regions_rows_exact(lib, n):
    """1..8 destinations, 1..4 columns with the key first or last: every destination's region holds exactly the rows (key
    and payload together) whose key maps to it (1,100,003 rows: more 4096-row tiles than the capped grid of 2 x 132 CTAs,
    so the CTAs loop).  Then the same rows with a bitmap on the key (at most 3 columns: the mask word is the 4th): a row
    whose key is NULL is neither counted nor sent"""
    rng = np.random.default_rng(n)
    keep = []
    try:
        for n_parts in range(1, 9):
            ncols = 1 + (n_parts - 1) % 4
            key_col = 0 if n_parts % 2 else ncols - 1
            cols = _push_data(rng, n, ncols, key_col, 0)
            ptrs = _dev_cols(lib, cols, keep)
            _push_one_source(lib, cols, ptrs, key_col, n_parts)
            nn = rng.random(n) >= 0.25
            bm = X.Buf(lib, ((n + 63) // 64) * 8 + 8, None)
            keep.append(bm)
            bm.put(X.bitmap_words(nn))
            m = min(ncols, 3)
            sub = slice(0, m) if key_col == 0 else slice(ncols - m, ncols)
            _push_one_source(lib, cols[sub], ptrs[sub], 0 if key_col == 0 else m - 1, n_parts, nn, bm.addr())
            for b in keep:
                b.free()
            keep.clear()
    finally:
        for b in keep:
            b.free()


def test_pushes_on_one_slot_keep_their_regions(lib):
    """two pushes on the same slot, into different regions with different caps and epochs, queued behind pushes that keep
    the push stream busy: the second call must not change where the first one scatters, its limits, or the slots it
    publishes to (the slot's staging is rewritten only after the previous push of that slot has read it).  The first push
    does not fit the second one's cap, so scattering under it would publish ~0."""
    rng = np.random.default_rng(8)
    keep, regs = [], []
    n_busy, n_parts, ncols = 1 << 25, 4, 2
    sizes = [200_003, 40_009]
    try:
        busy = rng.integers(-(1 << 63), (1 << 63) - 1, n_busy, dtype=np.int64)
        bptr = _dev_cols(lib, [busy], keep)
        data = [_push_data(rng, n, ncols, 0, i * sizes[0]) for i, n in enumerate(sizes)]
        ptrs = [_dev_cols(lib, d, keep) for d in data]
        dests = [X.push_dest(d[0], None, n_parts) for d in data]
        caps = [int(np.bincount(d, minlength=n_parts).max()) for d in dests]
        assert caps[0] > caps[1]
        dst = [X.Regions(lib, n_parts, ncols, cap) for cap in caps]
        regs += dst
        for s in range(4):                      # 1 GB of scatter stores queued on the push stream
            r = X.Regions(lib, 1, 1, n_busy, guard=8)
            regs.append(r)
            L.check(r.push(0, bptr, n_busy, s, 1))
        for i in range(2):
            L.check(dst[i].push(0, ptrs[i], sizes[i], 5, 2 + i))
        for s in (0, 1, 2, 3, 5):
            L.check(lib.tq_partition_push_sync(s))
        for i in range(2):
            _check_source(dst[i], 0, data[i], dests[i], 2 + i)
        assert regs[2].slots(0) == [(n_busy, 1)]
    finally:
        for b in keep + regs:
            b.free()


def test_push_regions_refusals(lib):
    """every bad argument: TQ_ERR_INVALID_ARG (more than 4 wire columns: TQ_ERR_UNSUPPORTED_TYPE), and no region, slot,
    miss column or miss slot is written; then the same buffers push correctly"""
    rng = np.random.default_rng(12)
    n, W, ncols = 5_000, 3, 2
    keep = []
    reg = X.Regions(lib, W, ncols, n)
    miss = X.Regions(lib, 1, ncols, n, GUARD)
    try:
        cols = _push_data(rng, n, ncols, 0, 0)
        tq = _tq(_dev_cols(lib, cols, keep), n)
        dest, cnts = reg.push_tables(0, 0)
        args = dict(n_cols=ncols, cols=tq, key_col=0, n=n, n_parts=W, selected=None, keep_misses=1, dest_data=dest, dest_counts=cnts,
                    region_cap=reg.cap[0], miss_data=miss.push_tables(0, 0)[0], miss_count=miss.slot_ptr(0, 0, 0), miss_cap=n, slot=0, epoch=1)
        push = lambda **bad: lib.tq_partition_push_regions(*{**args, **bad}.values())
        holes = [(C.c_void_p * len(a))(*a) for a in (dest, cnts)]      # the last destination without its last region / its count slot
        holes[0][len(dest) - 1] = holes[1][W - 1] = None
        for bad in (dict(n_parts=0), dict(n_parts=9), dict(n_parts=-1), dict(n=-1), dict(n=1 << 32), dict(key_col=-1),
                    dict(key_col=ncols), dict(n_cols=0), dict(cols=None), dict(dest_data=None), dict(dest_counts=None),
                    dict(dest_data=holes[0]), dict(dest_counts=holes[1]),
                    dict(slot=-1), dict(slot=16), dict(region_cap=0), dict(region_cap=1 << 32), dict(miss_data=None),
                    dict(miss_count=None), dict(miss_cap=-1), dict(miss_cap=1 << 32)):
            assert push(**bad) == L.TQ_ERR_INVALID_ARG, bad
        assert push(n_cols=5, cols=(L.TQColumn * 5)(*([tq[0]] * 5))) == L.TQ_ERR_UNSUPPORTED_TYPE
        for d in range(W):
            assert reg.slots(d) == [(0, 0)] * W, "a refused push published a slot"
            assert all(np.all(reg.region(d, 0, c) == X.SENTINEL) for c in range(ncols)), "a refused push wrote rows"
        assert miss.slots(0) == [(0, 0)], "a refused push published its miss slot"
        L.check(push())
        L.check(lib.tq_partition_push_sync(0))
        _check_source(reg, 0, cols, X.push_dest(cols[0], None, W), 1)
        assert miss.slots(0) == [(0, 1)], "no row misses: the miss slot reads {0, epoch}"
        assert all(np.all(miss.region(0, 0, c) == X.SENTINEL) for c in range(ncols)), "a miss column was written"
    finally:
        for b in keep + [reg, miss]:
            b.free()


def _shards(rng, sizes, ncols, first=0):
    out = []
    for n in sizes:
        out.append(_push_data(rng, n, ncols, 0, first))
        first += n
    return out


def _check_regions(reg, shards, epoch, overflowed=()):
    """slots and regions of every (destination, source) after the pushes of `shards` under `epoch`"""
    w = reg.world
    for s, cols in enumerate(shards):
        if s not in overflowed:
            _check_source(reg, s, cols, X.push_dest(cols[0], None, w), epoch)
            continue
        for d in range(w):
            assert reg.slots(d)[s] == ((1 << 64) - 1, epoch), f"source {s} overflowed: destination {d} must read ~0"
            got = np.stack([reg.region(d, s, c) for c in range(reg.ncols[0])], axis=1)
            assert np.all(got[reg.cap[0]:] == X.SENTINEL), f"region ({d}, {s}): a row past its cap"


def _push_all(lib, reg, shards, epoch, keep, slot0=0, wait=True):
    for s, cols in enumerate(shards):
        ptrs = _dev_cols(lib, cols, keep)
        L.check(reg.push(s, ptrs, len(cols[0]), slot0 + s, epoch))
    if wait:                                      # queued after the pushes that publish this epoch
        for d in range(reg.world):
            L.check(reg.wait(d, epoch))
    for s in range(len(shards)):
        L.check(lib.tq_partition_push_sync(slot0 + s))
    X.compute_sync(lib)


@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_push_regions_publish_and_wait(lib, W):
    """each emulated source s pushes its shard into its region on every destination (slot s), then publishes: a cap that is
    not a multiple of 4096, an exact fit, and one row short (that source's slots read ~0 everywhere, nothing lands past
    the cap).  The last source of W >= 2 has no rows and still publishes {0, epoch}."""
    rng = np.random.default_rng(W)
    ncols = 1 + W % 4
    sizes = [30_011 + 9_973 * s for s in range(W)]
    if W >= 2:
        sizes[-1] = 0
    shards = _shards(rng, sizes, ncols)
    cnt = np.array([np.bincount(X.push_dest(c[0], None, W), minlength=W) for c in shards])
    big = int(cnt.max())
    keep = []
    loose = big + 1000 + (1 if (big + 1000) % 4096 == 0 else 0)
    for epoch, cap in enumerate((loose, big, big - 1), start=3):
        reg = X.Regions(lib, W, ncols, cap)
        try:
            _push_all(lib, reg, shards, epoch, keep)
            over = {s for s in range(W) if cnt[s].max() > cap}
            assert len(over) == (1 if cap < big else 0)
            _check_regions(reg, shards, epoch, over)
        finally:
            reg.free()
            for b in keep:
                b.free()
            keep.clear()


def test_sixteen_push_slots_in_flight(lib):
    """two tables of 8 emulated ranks pushed on slots 0..7 and 8..15 before the first tq_partition_push_sync"""
    rng = np.random.default_rng(16)
    keep = []
    regs = [X.Regions(lib, 8, 2, 20_000), X.Regions(lib, 8, 3, 9_000)]
    try:
        shards = [_shards(rng, [60_000 + 1000 * s for s in range(8)], 2), _shards(rng, [40_000] * 8, 3, 1 << 30)]
        for t, reg in enumerate(regs):
            for s, cols in enumerate(shards[t]):
                L.check(reg.push(s, _dev_cols(lib, cols, keep), len(cols[0]), 8 * t + s, 7 + t))
        for slot in range(16):
            L.check(lib.tq_partition_push_sync(slot))
        for t, reg in enumerate(regs):
            _check_regions(reg, shards[t], 7 + t)
    finally:
        for b in keep + regs:
            b.free()


# ================================================================================================ C. segmented join
POS_LAUNCHES = 6        # probe launches of one batch on the streaming join's positional path


@pytest.fixture()
def _stream_partitions(monkeypatch):
    monkeypatch.setenv("TQ_JOIN_PART_ROWS", "4000")     # 128 partitions of the 300,000-row build side: the positional path
    monkeypatch.delenv("TQ_JOIN_NO_FAST", raising=False)


def _join_step(lib, reg, joins, shards, epoch, keep):
    """protocol order: every source's push, then per destination the device-side wait and the segmented batch, then the
    host waits for the pushes; the batch's rows are drained (which finalises it) before the regions are reused"""
    w = reg.world
    for s, cols in enumerate(shards):
        L.check(reg.push(s, _dev_cols(lib, cols, keep), len(cols[0]), s, epoch))
    for d in range(w):
        L.check(reg.wait(d, epoch))
        L.check(lib.tq_join_put_probe_segments(joins[d].h, w, reg.region_table(d, 0), reg.count_ptrs(d, 0), reg.cap[0]))
    for s in range(len(shards)):
        L.check(lib.tq_partition_push_sync(s))
    for j in joins:
        j.drain()
    X.compute_sync(lib)


@pytest.mark.parametrize("W", [2, 3, 8])
def test_segmented_join_over_pushed_regions(lib, W, _stream_partitions):
    """W destinations each join the W regions the sources pushed to them as one segmented batch; two steps on the same
    regions: step 1 with one source overflowing its cap (its regions read as empty everywhere), step 2 under epoch + 1 with
    fewer rows (the step-1 rows past the new counts must not come back).  The result of destination d is the oracle join
    of the rows sent to d, every key belongs to d, and together they are the join of every row that was not overflowed."""
    import test_gpu_stream_probe_columns as T
    rng = np.random.default_rng(50 + W)
    bcols = T._build_cols(rng, 2)
    bk = bcols[0].values
    keep, joins = [], []

    def shards(sizes, first):
        out = []
        for n in sizes:
            k = T._probe_keys(rng, bk, n, 0.1)
            out.append([k, np.arange(first, first + n, dtype=np.int64)])
            first += n
        return out
    s1 = shards([50_000 + 3_000 * s for s in range(W)], 0)
    s1[W - 1] = shards([150_000], 10_000_000)[0]              # the source that overflows in step 1
    s2 = shards([20_000 + 1_000 * s for s in range(W)], 20_000_000)
    cnt1 = np.array([np.bincount(X.push_dest(c[0], None, W), minlength=W) for c in s1])
    cap = int(cnt1[:W - 1].max()) + 17
    assert cnt1[W - 1].max() > cap
    reg = X.Regions(lib, W, 2, cap, guard=4096)       # the join reads regions in whole 4096-row tiles
    try:
        joins = [T._Join(lib, bcols, 2) for _ in range(W)]
        assert all(j.parts == 128 for j in joins), "the build did not take 128 partitions"
        launches0 = [j.stats()[7] for j in joins]
        _join_step(lib, reg, joins, s1, 1, keep)
        assert all(reg.slots(d)[W - 1][0] == (1 << 64) - 1 for d in range(W))
        _join_step(lib, reg, joins, s2, 2, keep)
        sent = [c for c in s1[:W - 1]] + s2
        everything = []
        for d, j in enumerate(joins):
            got, st = j.finish()
            assert st[7] - launches0[d] == 2 * POS_LAUNCHES, "a segmented batch left the positional path"
            mine = [np.concatenate([c[i][X.push_dest(c[0], None, W) == d] for c in sent]) for i in range(2)]
            want = T._want(bcols, mine)
            assert_same_multiset(got, want)
            if got.num_rows():
                assert np.all(dest_rank_np(got.cols[0].values, W) == d), "a key joined on the wrong destination"
            everything.append(got)
        allp = [np.concatenate([c[i] for c in sent]) for i in range(2)]
        from tinysql_b200.chunk import Chunk
        assert_same_multiset(Chunk.concat(everything, [INT64] * 4), T._want(bcols, allp))
    finally:
        for j in joins:
            j.close()
        reg.free()
        for b in keep:
            b.free()


def test_segmented_join_segment_limit(lib, _stream_partitions):
    """8 segments (SA_MAX_SEGS) are one batch; 9 are refused before anything is read"""
    import test_gpu_stream_probe_columns as T
    rng = np.random.default_rng(9)
    bcols = T._build_cols(rng, 2)
    bk = bcols[0].values
    keep = []
    reg = X.Regions(lib, 9, 2, 8_192, guard=4096)
    j = T._Join(lib, bcols, 2)
    try:
        sh = [[T._probe_keys(rng, bk, 5_000, 0.1), np.arange(5_000 * s, 5_000 * (s + 1), dtype=np.int64)] for s in range(8)]
        for s, cols in enumerate(sh):       # 8 sources into destination 0's regions of a 9-rank table (n_parts = 1: its entries come first)
            ptrs = _dev_cols(lib, cols, keep)
            dest, cnts = reg.push_tables(0, s)
            L.check(lib.tq_partition_push_regions(2, _tq(ptrs, 5_000), 0, 5_000, 1, None, 0, dest, cnts, reg.cap[0], None, None, 0, s, 1))
        for s in range(8):
            L.check(lib.tq_partition_push_sync(s))
        cols, cnts = reg.region_table(0, 0), reg.count_ptrs(0, 0)
        assert lib.tq_join_put_probe_segments(j.h, 9, cols, cnts, reg.cap[0]) == L.TQ_ERR_INVALID_ARG
        L.check(lib.tq_join_put_probe_segments(j.h, 8, cols, cnts, reg.cap[0]))
        got, _ = j.finish()
        assert_same_multiset(got, T._want(bcols, [np.concatenate([c[i] for c in sh]) for i in range(2)]))
    finally:
        j.close()
        reg.free()
        for b in keep:
            b.free()


# ================================================================================================ D. dist.py on the device
def _exchange_in_process(parts, world):
    """what the NCCL all-to-all delivers: destination d receives every source's slice [off[d], off[d + 1]) per column"""
    import torch
    return [[torch.cat([cols[c][off[d]:off[d + 1]] for cols, off in parts]) for c in range(len(parts[0][0]))] for d in range(world)]


@pytest.mark.parametrize("W", [2, 3, 8])
def test_distributed_group_by_and_join(lib, W):
    """dist.gpu_agg_fns / gpu_partition_fn / gpu_local_join with W emulated ranks: integer COUNT / SUM / AVG / MAX / MIN
    equal the oracle over all rows, every group is finalised once, on dest_rank_np(key); a FLOAT64 GROUP BY key that is
    +0.0 on some shards and -0.0 on others is one group; the partitioned join is the oracle join"""
    import torch

    from tinysql_b200 import dist as D
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(60 + W)
    part = D.gpu_partition_fn(lib, L)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    # ---- GROUP BY an int key and a FLOAT64 key
    for key_tp in (INT64, FLOAT64):
        n_s = [40_000 + 777 * s for s in range(W)]
        if key_tp == INT64:
            keys = [rng.integers(-3000, 3000, n).astype(np.int64) for n in n_s]
            keys[0][:5] = [np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1, X.EMPTY_KEY.view(np.int64)]
        else:
            keys = [rng.integers(-200, 200, n) * 0.5 for n in n_s]
            for s in range(W):
                keys[s][:50] = -0.0 if s % 2 else 0.0
        vals = [rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64) for n in n_s]
        funcs = [(5, 0), (0, -1), (1, 1), (2, 1), (3, 1), (4, 1)]      # FIRSTROW(k) COUNT(*) SUM(v) AVG(v) MAX(v) MIN(v)
        pfn, ffn = D.gpu_agg_fns(lib, L, [key_tp, INT64], 0, funcs, est_groups=8192)
        parts = [part(pfn([t(keys[s]), t(vals[s])]), W) for s in range(W)]
        got = []
        for d, recv in enumerate(_exchange_in_process(parts, W)):
            res = ffn(recv)
            if res[0].length:
                assert np.all(dest_rank_np(res[0].raw().view(np.int64), W) == d), "a group was finalised on the wrong rank"
                got.append(np.stack([c.raw() for c in res], axis=1))
        got = np.concatenate(got)
        K, V = np.concatenate(keys), np.concatenate(vals)
        rc, want = O.hash_agg([key_tp, INT64], [Column(key_tp, K), Column(INT64, V)], [0], funcs)
        wantm = np.stack([c.raw() for c in want.cols], axis=1)
        assert rc == 0
        assert len(np.unique(got[:, 0])) == len(got), "a group was finalised on more than one rank"
        if key_tp == FLOAT64:
            zeros = got[:, 0][np.abs(got[:, 0].view(np.float64)) == 0.0]
            assert len(zeros) == 1, f"+0.0 and -0.0 made {len(zeros)} groups"
            got[:, 0] = np.where(got[:, 0] == np.float64(-0.0).view(np.uint64), np.uint64(0), got[:, 0])
            wantm[:, 0] = np.where(wantm[:, 0] == np.float64(-0.0).view(np.uint64), np.uint64(0), wantm[:, 0])
        assert got.shape == wantm.shape, (got.shape, wantm.shape)
        assert np.array_equal(X.sorted_rows(got), X.sorted_rows(wantm)), f"distributed GROUP BY ({key_tp}) differs from the oracle"
    # ---- join: both sides partitioned by key, each destination joins what it received
    nb, npr = 60_000, 150_000
    bk = rng.permutation(nb * W).astype(np.int64) * 5 - 7
    bsh = np.array_split(bk, W)
    psh = [rng.choice(bk, npr) + (rng.random(npr) < 0.1) for _ in range(W)]     # ~10 % misses (key + 1)
    bparts = [part([t(b), t(b * 3 + 1)], W) for b in bsh]
    pparts = [part([t(p), t(np.arange(npr, dtype=np.int64) + s * npr)], W) for s, p in enumerate(psh)]
    out = []
    for d, (b, p) in enumerate(zip(_exchange_in_process(bparts, W), _exchange_in_process(pparts, W))):
        rows, _, res = D.gpu_local_join(lib, L, b, p, keep_result=True)
        if rows:
            m = np.stack([c.values for c in res], axis=1)
            assert len(m) == rows, "the join's result came in several batches and only the last was kept"
            assert np.all(dest_rank_np(m[:, 0], W) == d)
            out.append(m)
    got = np.concatenate(out)
    P = np.concatenate(psh)
    want = O.hash_join(0, True, [INT64, INT64], [Column(INT64, bk), Column(INT64, bk * 3 + 1)], [INT64, INT64],
                       [Column(INT64, P), Column(INT64, np.arange(W * npr, dtype=np.int64))], [0], [0])
    wantm = np.stack([c.values for c in want.cols], axis=1)
    assert np.array_equal(X.sorted_rows(got.view(np.uint64)), X.sorted_rows(wantm.view(np.uint64)))
