"""Multi-GPU hash join and GROUP BY: radix-partition the rows (the join's) or the partial groups (the GROUP BY's) on the key
across the ranks, exchange the partitions, run the single-GPU operator on what arrived.  One process per GPU;
torch.distributed is plumbing only (process group, barriers, the NCCL variant); partitioning, exchange, join and aggregation
are the CUDA kernels of libtinysql_b200.so.

Two exchanges:
  * RegionExchange: the scatter kernel stores every row straight into the destination rank's receive region over NVLink peer
    memory (CUDA IPC); device-side epoch flags replace host barriers.
      - RegionJoin (the default of bench.py --gpus N): chunk by chunk, overlapped with the local join of the chunks that have
        already arrived.
      - BroadcastJoin: every rank copies its build shard to every rank (tq_partition_push_broadcast) and joins its own probe
        shard in place; runs every join the single-GPU handle runs (key-less, multi-column and string keys, wide rows,
        OtherConditions).  Use it where RegionJoin cannot route the join, or where the build side is small: it moves
        (W-1) x the build side over NVLink and holds W x the build side per rank, where the shuffle moves (W-1)/W of both
        sides.  RegionJoin stays the path for the one-key joins it runs.
      - RegionAgg: each rank's Partial1 aggregation pushes its partial rows (tq_agg_push_partial, NULL mask word included, any
        number of GROUP BY items) to the rank its group names; that rank merges the regions in place
        (tq_agg_merge_regions) and finalises.
  * exchange() (distributed_join / distributed_agg): partition locally, then ONE grouped NCCL send/recv — the all-to-all at the
    shard boundary (NCCL 2.27/2.28 has no ncclAllToAllv); also what the gloo CPU tests drive.  distributed_agg takes one
    NOT NULL GROUP BY item.

The moral equivalent of the reference's partial->final hash shuffle (executor/aggregate.go:96-133,352-356): a row goes to
rank  (mix64(key) >> 40) % world  — a pure function of its key, so equal keys meet on one rank and nothing else moves.

The exchange logic is backend-agnostic (gloo on CPU in tests/test_dist_gloo.py with injected partition / join functions).
"""
import ctypes as C
import os
import time

import numpy as np
import torch
import torch.distributed as dist


def mix64_np(k):
    """tqd::mix64 (csrc/common.cuh) in numpy, for the CPU stand-in partitioner of the gloo tests."""
    k = k.astype(np.uint64).copy()
    k ^= k >> np.uint64(33)
    k *= np.uint64(0xFF51AFD7ED558CCD)
    k ^= k >> np.uint64(33)
    k *= np.uint64(0xC4CEB9FE1A85EC53)
    k ^= k >> np.uint64(33)
    return k


def dest_rank_np(keys, world):
    return ((mix64_np(keys) >> np.uint64(40)) % np.uint64(world)).astype(np.int64)


def exchange_counts(send_offsets_list, world, rank, device, group=None):
    """One all-gather for any number of partitioned tables: returns, per table, the rows every source rank sends HERE."""
    mine = torch.tensor([[offs[p + 1] - offs[p] for p in range(world)] for offs in send_offsets_list], dtype=torch.int64, device=device)
    allc = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(allc, mine, group=group)            # world x tables x world counts (tiny)
    m = torch.stack(allc).cpu().numpy()                 # ONE device->host sync
    return [[int(m[src, t, rank]) for src in range(world)] for t in range(len(send_offsets_list))]


def exchange(cols, send_offsets, world, rank, group=None, recv_counts=None, async_op=False):
    """cols: list of 1-D tensors, all partitioned the same way: rows [send_offsets[p], send_offsets[p+1]) go to rank p.
    Returns (list of received columns, recv_counts[, work handles]).  NCCL: one all_to_all_single per column (NCCL
    send/recv groups inside); other backends (gloo has no all-to-all): one grouped batch of isend/irecv."""
    dev = cols[0].device
    if recv_counts is None:
        recv_counts = exchange_counts([send_offsets], world, rank, dev, group)[0]
    send_counts = [int(send_offsets[p + 1] - send_offsets[p]) for p in range(world)]
    total = int(sum(recv_counts))
    out = [torch.empty(total, dtype=c.dtype, device=dev) for c in cols]
    works = []
    if dist.get_backend(group) == "nccl":
        for ci, c in enumerate(cols):
            src = c[int(send_offsets[0]): int(send_offsets[world])]
            w = dist.all_to_all_single(out[ci], src, output_split_sizes=recv_counts, input_split_sizes=send_counts, group=group, async_op=async_op)
            if async_op:
                works.append(w)
    else:
        recv_off = np.concatenate([[0], np.cumsum(recv_counts)]).astype(np.int64)
        ops = []
        for ci, c in enumerate(cols):
            for peer in range(world):
                s_lo, s_hi = int(send_offsets[peer]), int(send_offsets[peer + 1])
                r_lo, r_hi = int(recv_off[peer]), int(recv_off[peer + 1])
                if peer == rank:
                    out[ci][r_lo:r_hi].copy_(c[s_lo:s_hi])
                    continue
                if s_hi > s_lo:
                    ops.append(dist.P2POp(dist.isend, c[s_lo:s_hi], peer, group=group))
                if r_hi > r_lo:
                    ops.append(dist.P2POp(dist.irecv, out[ci][r_lo:r_hi], peer, group=group))
        if ops:
            for req in dist.batch_isend_irecv(ops):  # one group around every send and recv
                req.wait()
    if async_op:
        return out, recv_counts, works
    return out, recv_counts


class RawCol:
    """a device column that is just (pointer, rows): quacks like the torch tensors the helpers below take"""

    def __init__(self, ptr, n):
        self.ptr, self.n = ptr, n

    def data_ptr(self):
        return self.ptr

    def numel(self):
        return self.n

    def __getitem__(self, sl):
        assert sl.start in (None, 0) and sl.step in (None, 1)
        return RawCol(self.ptr, min(self.n, sl.stop))


def _round_up(x, m):
    return (x + m - 1) // m * m


class RegionLayout:
    """Where the region exchange's slots and regions sit in a destination's receive buffer, and the argument tables the C
    calls take from them.  tables = [(wire columns, cap rows)] per table t, or (wire columns, cap rows, [words per wire
    column]) for a table whose areas are not cap rows of 8 bytes each (the broadcast's offsets, cells and bitmap words);
    every destination's buffer (bytes long, at bases[d], set by whoever places the buffers) holds

        slot[t][src]        = {u64 rows, u64 epoch}             16 bytes per (table, source), from offset 0
        region[t][src][c]   = cap_t rows x 8 bytes              from the first page boundary after the slots

    with pad_rows rows (words) left unused after every region (0 in production; the emulated-rank tests fill them with a sentinel,
    so a row written past the cap lands inside the allocation).  bytes is page-aligned, so receive buffers placed back to
    back keep their slot blocks page-aligned.  Needs no process group, no IPC and no torch: RegionExchange places it over
    the IPC-opened buffers of the ranks, RegionJoin over one local buffer for its kept miss rows, the tests over W
    emulated ranks in one allocation."""

    def __init__(self, lib, L, world, tables, pad_rows=0):
        self.lib, self.L, self.world, self.pad_rows = lib, L, world, pad_rows
        self.ncols = [t[0] for t in tables]
        self.cap = [int(t[1]) for t in tables]
        # words per wire column: cap, unless the table lists its own (nc, cap, [words per wire column]) — the broadcast's
        # offsets, cells and bitmap words; every column is followed by pad_rows words
        self.col_off, self.stride, self.reg_off = [], [], []
        for t, cap in zip(tables, self.cap):
            words = [int(x) for x in t[2]] if len(t) > 2 else [cap] * t[0]
            self.col_off.append([sum(words[:c]) + c * pad_rows for c in range(len(words))])
            self.stride.append(sum(words) + len(words) * pad_rows)
        off = _round_up(len(tables) * world * 16, 4096)
        for stride in self.stride:
            self.reg_off.append(off)
            off += world * stride * 8
        self.bytes = _round_up(off, 4096)
        self.bases = []

    def region_ptr(self, dst, t, src, c):
        return self.bases[dst] + self.reg_off[t] + (src * self.stride[t] + self.col_off[t][c]) * 8

    def slot_ptr(self, dst, t, src):
        return self.bases[dst] + (t * self.world + src) * 16

    def push_tables(self, t, src):
        """(dest_data, dest_counts) of source src for table t, as tq_partition_push_regions and tq_agg_push_partial take them:
        dest_data[q * nw + c] = its region of wire column c on destination q, dest_counts[q] = its slot there"""
        w, nw = self.world, self.ncols[t]
        dest = (C.c_void_p * (w * nw))(*[self.region_ptr(q, t, src, c) for q in range(w) for c in range(nw)])
        return dest, (C.c_void_p * w)(*[self.slot_ptr(q, t, src) for q in range(w)])

    def region_table(self, dst, t):
        """destination dst's regions of table t as tq_column [src][col] (length = cap), as tq_region_gather,
        tq_agg_merge_regions and tq_join_put_probe_segments take them"""
        w, nw = self.world, self.ncols[t]
        regs = (self.L.TQColumn * (w * nw))()
        for k in range(w * nw):
            regs[k].length, regs[k].data = self.cap[t], self.region_ptr(dst, t, k // nw, k % nw)
        return regs

    def count_ptrs(self, dst, t):
        """the slot of every source on destination dst for table t (tq_join_put_probe_segments)"""
        return (C.c_void_p * self.world)(*[self.slot_ptr(dst, t, g) for g in range(self.world)])

    def read_slots(self, dst, t0=0, nt=None):
        """one host read of destination dst's slots of tables t0 .. t0 + nt - 1 (every table from t0 by default): uint64 array
        [table][src][rows, epoch]"""
        raw = np.zeros((len(self.cap) - t0 if nt is None else nt, self.world, 2), np.uint64)
        self.L.check(self.lib.tq_memcpy_d2h(raw.ctypes.data, C.c_void_p(self.slot_ptr(dst, t0, 0)), raw.nbytes))
        return raw

    def counts(self, dst, t0=0, nt=None):
        """rows every source published on destination dst, per table (read_slots); a count past its table's cap (an overflowed
        push publishes ~0: it dropped rows) raises RuntimeError"""
        out = []
        for t, raw in enumerate(self.read_slots(dst, t0, nt), start=t0):
            cnt = [int(r) for r in raw[:, 0]]
            if any(c > self.cap[t] for c in cnt):
                raise RuntimeError(f"region overflow in table {t}: {cnt} rows, capacity {self.cap[t]} (skewed keys)")
            out.append(cnt)
        return out


class RegionExchange(RegionLayout):
    """The exchange the multi-GPU join and GROUP BY run on: a RegionLayout over one device allocation per rank
    (tq_device_alloc, exported once through CUDA IPC and opened by every peer under its own device); caps are rounded up to
    align_rows.  A rank pushes table t with tq_partition_push_regions: its scatter kernel stores rows straight into "its"
    region on every peer (NVLink peer stores, no staging, no count exchange first) and then publishes count + epoch in the
    peer's slot.  The receiver enqueues tq_region_wait(slots[t], world, epoch) — a device-side wait — in front of the
    kernels that read the regions and joins them as one segmented batch (tq_join_put_probe_segments): no host round trip
    and no NCCL call sits between the exchange and the join."""

    def __init__(self, lib, L, world, rank, tables, align_rows=4096):
        super().__init__(lib, L, world, [(t[0], _round_up(t[1], align_rows)) + tuple(t[2:]) for t in tables])
        self.rank = rank
        p = C.c_void_p()
        L.check(lib.tq_device_alloc(self.bytes, C.byref(p)))
        L.check(lib.tq_memset_device(p, 0, self.bytes))
        L.check(lib.tq_device_synchronize())
        self.own = p.value
        h = (C.c_ubyte * 64)()
        L.check(lib.tq_ipc_get_handle(p, h))
        gathered = [None] * world
        dist.all_gather_object(gathered, bytes(h))
        self._opened = []
        for d in range(world):
            if d == rank:
                self.bases.append(self.own)
                continue
            q = C.c_void_p()
            buf = (C.c_ubyte * 64).from_buffer_copy(gathered[d])
            L.check(lib.tq_ipc_open_handle(buf, C.byref(q)))
            self.bases.append(q.value)
            self._opened.append(q.value)
        self.epoch = 0

    def close(self):
        for p in self._opened:
            self.lib.tq_ipc_close_handle(C.c_void_p(p))
        self._opened = []
        dist.barrier()  # nobody frees a buffer a peer still has mapped
        self.lib.tq_device_free(C.c_void_p(self.own))

    def next_epoch(self):
        self.epoch += 1
        return self.epoch

    def push(self, t, cols, n, slot, bitmaps=None, selected=None, miss=None):
        """scatter this rank's rows of table t into its region on every rank; asynchronous (push stream).  bitmaps: a device
        NULL bitmap pointer (or None) per column; with any, the mask word travels as table t's last wire column.  selected:
        device address of n bytes (0/1) or None.  miss: (RegionLayout of one destination, its table) that keeps the rows
        which cannot match on this rank, or None to drop them."""
        arr = _tq_cols(self.L, cols, n)
        for c, b in enumerate(bitmaps or []):
            arr[c].null_bitmap = b
        dest, cnts = self.push_tables(t, self.rank)
        miss_cols, miss_slot, miss_cap = None, None, 0
        if miss is not None:
            ml, mt = miss
            miss_cols, miss_slot, miss_cap = ml.push_tables(mt, 0)[0], ml.slot_ptr(0, mt, 0), ml.cap[mt]
        self.L.check(self.lib.tq_partition_push_regions(len(cols), arr, 0, n, self.world, selected, int(miss is not None), dest, cnts, self.cap[t],
                                                        miss_cols, miss_slot, miss_cap, slot, self.epoch))

    def wait(self, t):
        """device-side: the compute stream waits until every source has published table t for this epoch"""
        self.L.check(self.lib.tq_region_wait(C.c_void_p(self.slot_ptr(self.rank, t, 0)), self.world, self.epoch))


def distributed_join(build_cols, probe_cols, world, rank, partition_fn, local_join_fn, group=None):
    """build_cols / probe_cols: lists of tensors holding this rank's row shard; key = column 0 of each side.
    partition_fn(cols, world) -> (partitioned cols, offsets[world+1]);  local_join_fn(build, probe) -> result."""
    b_part, b_off = partition_fn(build_cols, world)
    b_recv, _ = exchange(b_part, b_off, world, rank, group)
    p_part, p_off = partition_fn(probe_cols, world)
    p_recv, _ = exchange(p_part, p_off, world, rank, group)
    return local_join_fn(b_recv, p_recv)


def distributed_agg(cols, world, rank, partial_fn, partition_fn, final_fn, group=None):
    """The reference's partial -> shuffle -> final HashAgg (executor/aggregate.go:96-133,352-356,424-457) across ranks:
    partial_fn(cols) -> partial rows as a list of int64 tensors, GROUP BY key first (one row per LOCAL group:
    rows/world -> <= NDV rows, so the exchange moves groups, not input rows); partition_fn as in distributed_join
    (same key -> rank rule); final_fn(received partial rows) -> this rank's final groups (MergePartialResult)."""
    partials = partial_fn(cols)
    part, off = partition_fn(partials, world)
    recv, _ = exchange(part, off, world, rank, group)
    return final_fn(recv)


# ---------------------------------------------------------------------------------------------- GPU plumbing
def gpu_agg_fns(lib, L, types, group_col, funcs, est_groups=0):
    """(partial_fn, final_fn) for distributed_agg on device-resident NOT NULL int64/float64 columns: Partial1 handle ->
    tq_agg_export_partial; Final handle <- tq_agg_merge_partial.  Columns are declared TQ_TYPE_NOT_NULL: the partial
    states then carry no NULLs, so the exchange moves plain 8-byte columns (nullable inputs: merge locally instead)."""
    def make():
        it = (C.c_int32 * len(types))(*[t | L.TQ_TYPE_NOT_NULL for t in types])
        gb = (C.c_int32 * 1)(group_col)
        fa = (L.TQAggFunc * len(funcs))(*[L.TQAggFunc(f, a) for f, a in funcs])
        d = L.TQAggDesc(len(types), it, 1, gb, len(funcs), fa, est_groups)
        h = C.c_void_p()
        L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
        return h, (it, gb, fa)

    def partial_fn(cols):
        torch.cuda.synchronize()   # the library works on its own stream
        h, keep = make()
        try:
            n = int(cols[0].numel())
            if n:
                L.check(lib.tq_agg_put(h, _tq_cols(L, cols, n), L.TQ_MEM_DEVICE))
            width = C.c_int32(0)
            L.check(lib.tq_agg_partial_width(h, C.byref(width)))
            out = (L.TQColumn * width.value)()
            rows = C.c_int64(0)
            L.check(lib.tq_agg_export_partial(h, out, C.byref(rows)))
            # the lent arrays die with the handle: copy them into tensors the exchange can own
            res = []
            for c in range(width.value):
                t = torch.empty(rows.value, dtype=torch.int64, device=cols[0].device)
                if rows.value:
                    torch.cuda.current_stream().synchronize()
                    L.check(lib.tq_memcpy_d2d(t.data_ptr(), out[c].data, rows.value * 8))
                res.append(t)
        finally:
            lib.tq_agg_destroy(h)
        return res

    def final_fn(recv):
        torch.cuda.synchronize()
        h, keep = make()
        try:
            n = int(recv[0].numel())
            if n:
                L.check(lib.tq_agg_merge_partial(h, _tq_cols(L, recv, n), L.TQ_MEM_DEVICE))
            L.check(lib.tq_agg_eof(h))
            out = (L.TQColumn * len(funcs))()
            rows, eof = C.c_int64(0), C.c_int32(0)
            L.check(lib.tq_agg_next_device(h, out, C.byref(rows), C.byref(eof)))
            from .chunk import device_to_host
            res = []
            for i in range(len(funcs)):
                t = C.c_int32(0)
                L.check(lib.tq_agg_output_type(h, i, C.byref(t)))
                res.append(device_to_host(t.value, out[i].data, out[i].null_bitmap, rows.value))
        finally:
            lib.tq_agg_destroy(h)
        return res
    return partial_fn, final_fn


def _tq_cols(L, tensors, n):
    arr = (L.TQColumn * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i].length, arr[i].data, arr[i].null_bitmap, arr[i].offsets = n, t.data_ptr(), None, None
    return arr


def gpu_partition_fn(lib, L):
    def fn(cols, world):
        n = int(cols[0].numel())
        out = [torch.empty_like(c) for c in cols]
        offs = (C.c_int64 * (world + 1))()
        types = (C.c_int32 * len(cols))(*([1] * len(cols)))
        torch.cuda.synchronize()
        L.check(lib.tq_partition_device(len(cols), _tq_cols(L, cols, n), types, 0, n, world, _tq_cols(L, out, n), offs))
        return out, list(offs)
    return fn


def join_begin(lib, L, build, n_probe_cols=2):
    """create the join and build its table from device-resident build columns (key = column 0)"""
    nb = int(build[0].numel())
    t_b = (C.c_int32 * len(build))(*([1] * len(build)))
    t_p = (C.c_int32 * n_probe_cols)(*([1] * n_probe_cols))
    k = (C.c_int32 * 1)(0)
    d = L.TQJoinDesc(0, 1, len(build), t_b, n_probe_cols, t_p, 1, k, k, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    try:
        if nb:
            L.check(lib.tq_join_put_build(h, _tq_cols(L, build, nb), L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
    except Exception:
        lib.tq_join_destroy(h)
        raise
    return (h, len(build))


def join_finish(lib, L, handle, probe, keep_result=False):
    """probe with device-resident columns, drain, destroy.  Returns (rows, stats[, columns])."""
    h, n_build_cols = handle
    npr = int(probe[0].numel())
    total = 0
    result = None
    try:
        if npr:
            L.check(lib.tq_join_put_probe(h, _tq_cols(L, probe, npr), None, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_probe_eof(h))
        out = (L.TQColumn * (n_build_cols + len(probe)))()
        n, eof = C.c_int64(0), C.c_int32(0)
        while True:
            L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
            if n.value == 0 and eof.value:
                break
            total += n.value
            if keep_result and n.value:
                from .chunk import device_to_host
                result = [device_to_host(1, out[c].data, None, n.value) for c in range(n_build_cols + len(probe))]
        st = (C.c_int64 * 8)()
        lib.tq_join_stats(h, st)
    finally:
        lib.tq_join_destroy(h)
    return (total, list(st), result) if keep_result else (total, list(st))


def gpu_local_join(lib, L, build, probe, keep_result=False):
    """inner join, key = column 0 of both sides, int64 columns, inputs resident in HBM."""
    return join_finish(lib, L, join_begin(lib, L, build, len(probe)), probe, keep_result)


class RegionJoin:
    """The multi-GPU join over a RegionExchange.  Tables: 0 = build side, 1 + c = probe chunk c.  One step:

        push stream    push(build) | push(chunk 0) | push(chunk 1) | ...        (all enqueued up front; NVLink stays busy)
        compute stream wait(build) -> local build | wait(chunk 0) -> join | wait(chunk 1) -> join | ...

    wait(t) is the device-side tq_region_wait; the chunk-c join overlaps the chunk-(c+1) push.  Host synchronisation: one count
    read for the build side (tq_join_put_build takes host lengths), the result drain, and ONE barrier at the end of the step
    (nobody may overwrite a region a peer is still joining).

    The join is an ordinary tq_join_desc with the key in column 0 of both sides: join_type / outer_is_right as on one GPU,
    INT64 / UINT64 / FLOAT64 columns, optional defaultInner.  An inner join of NOT NULL columns reads the regions in place
    (tq_join_put_probe_segments).  Otherwise (an outer join, or a side declared nullable) a nullable side's push carries the
    mask word, the probe rows of an outer join that cannot match (NULL key, selected == 0) stay on this rank, and the
    receiver copies each table's regions into contiguous columns with tq_region_gather before tq_join_put_build /
    tq_join_put_probe; the kept rows are one more probe batch, unselected.  They land in a local RegionLayout of one
    destination (one table per probe chunk), so _gather reads them as it reads the exchanged tables."""

    def __init__(self, lib, L, world, rank, n_build_max, n_probe_max, n_chunks, slack=1.25, join_type=0, outer_is_right=True,
                 build_types=None, probe_types=None, build_nullable=False, probe_nullable=False, default_inner=None):
        """n_build_max / n_probe_max: the largest per-rank shard (every rank must pass the same numbers: the layout is shared).
        build_types / probe_types: TQ_TYPE_* per column (default two INT64 columns).  *_nullable: that side may carry NULL
        bitmaps.  default_inner: the inner side of a miss row, one value (int or float) or None per build column."""
        self.lib, self.L, self.world, self.rank, self.n_chunks = lib, L, world, rank, n_chunks
        self.join_type, self.outer_is_right = join_type, bool(outer_is_right)
        self.build_types = list(build_types or (L.TQ_TYPE_INT64, L.TQ_TYPE_INT64))
        self.probe_types = list(probe_types or (L.TQ_TYPE_INT64, L.TQ_TYPE_INT64))
        self.default_inner = default_inner
        self.bmask, self.pmask = int(bool(build_nullable)), int(bool(probe_nullable))
        self.segmented = join_type == 0 and not build_nullable and not probe_nullable
        nb, npc = len(self.build_types), len(self.probe_types)
        cap = lambda n: int(n / world * slack) + (1 << 14)   # keys are hash-spread: +25 % covers the imbalance between (source, destination) pairs
        # the gather path cuts a nullable probe side at whole 64-row bitmap groups: a chunk may be up to 63 rows longer
        self.chunk_max = (n_probe_max + n_chunks - 1) // n_chunks + (0 if self.segmented else 64)
        tables = [(nb + self.bmask, cap(n_build_max))] + [(npc + self.pmask, cap(self.chunk_max)) for c in range(n_chunks)]
        self.rx = RegionExchange(lib, L, world, rank, tables)
        self._bufs = []
        self.outer = join_type != 0
        if not self.segmented:
            rx = self.rx
            # receive side: the build table and one probe chunk as contiguous columns (+ bitmaps), and the kept miss rows
            self.g_build = self._cols(nb, world * rx.cap[0], self.bmask)
            self.g_probe = self._cols(npc, world * rx.cap[1], self.pmask)
            if self.outer:
                self.g_miss = self._cols(npc, self.chunk_max, self.pmask)
                self.misses = RegionLayout(lib, L, 1, [(npc + self.pmask, self.chunk_max)] * n_chunks)
                self.misses.bases = [self._alloc(self.misses.bytes, zero=True)]

    def _alloc(self, nbytes, zero=False):
        p = C.c_void_p()
        self.L.check(self.lib.tq_device_alloc(nbytes, C.byref(p)))
        self._bufs.append(p.value)
        if zero:
            self.L.check(self.lib.tq_memset_device(p, 0, nbytes))
            self.L.check(self.lib.tq_device_synchronize())
        return p.value

    def _ones(self, n):
        """a device NOT-NULL-everywhere bitmap of at least n rows"""
        if getattr(self, "_ones_rows", 0) < n:
            nbytes = ((n + 63) // 64) * 8 + 8
            self._ones_ptr, self._ones_rows = self._alloc(nbytes), n
            self.L.check(self.lib.tq_memset_device(C.c_void_p(self._ones_ptr), 0xFF, nbytes))
            self.L.check(self.lib.tq_device_synchronize())
        return self._ones_ptr

    def _cols(self, ncols, rows, nullable):
        """ncols device columns of `rows` rows for tq_region_gather, with device bitmaps when nullable"""
        arr = (self.L.TQColumn * ncols)()
        for c in range(ncols):
            arr[c].data = self._alloc(max(rows, 1) * 8)
            arr[c].null_bitmap = self._alloc(((rows + 63) // 64) * 8 + 8) if nullable else None
        return arr, rows

    def close(self):
        self.rx.close()
        for p in self._bufs:
            self.lib.tq_device_free(C.c_void_p(p))
        self._bufs = []

    def _desc(self):
        L = self.L
        tb = (C.c_int32 * len(self.build_types))(*self.build_types)
        tp = (C.c_int32 * len(self.probe_types))(*self.probe_types)
        k = (C.c_int32 * 1)(0)
        dbits = dnn = None
        if self.default_inner is not None:
            vals = [0 if v is None else int(np.array([v], dtype=np.float64 if t == L.TQ_TYPE_FLOAT64 else (np.uint64 if t == L.TQ_TYPE_UINT64 else np.int64)).view(np.uint64)[0])
                    for v, t in zip(self.default_inner, self.build_types)]
            dbits = (C.c_uint64 * len(vals))(*vals)
            dnn = (C.c_uint8 * len(vals))(*[0 if v is None else 1 for v in self.default_inner])
        d = L.TQJoinDesc(self.join_type, 1 if self.outer_is_right else 0, len(self.build_types), tb, len(self.probe_types), tp, 1, k, k, 0, 0,
                         C.cast(dbits, C.POINTER(C.c_uint64)) if dbits is not None else None, C.cast(dnn, C.POINTER(C.c_uint8)) if dnn is not None else None)
        return d, (tb, tp, k, dbits, dnn)

    def step(self, bk, bv, pk, pv, keep_result=False):
        """bk / bv / pk / pv: this rank's row shards as (device pointer, rows)-like objects.  Returns (rows, stats, result)."""
        return self.step_cols([bk, bv], [pk, pv], keep_result=keep_result)

    def step_cols(self, build, probe, build_bitmaps=None, probe_bitmaps=None, selected=None, keep_result=False):
        """build / probe: this rank's shard of every column ((device pointer, rows)-like objects, key = column 0).
        *_bitmaps: a device NULL bitmap pointer (or None) per column, on a side declared nullable.  selected: device bytes
        (0/1, one per probe row: the outer-side filter) or None.  Returns (rows, stats, result); result (keep_result) is a
        list of numpy value arrays on the segmented path, of host chunk Columns (with their NULLs) otherwise."""
        lib, L, rx, w = self.lib, self.L, self.rx, self.world
        if self.segmented and (build_bitmaps or probe_bitmaps or selected is not None):
            raise ValueError("RegionJoin: NULL bitmaps need build_nullable / probe_nullable, selected[] an outer join")
        t_start = time.perf_counter()
        trace = []
        mark = lambda name: trace.append((name, (time.perf_counter() - t_start) * 1e3))   # host-side timeline: where the host blocks
        n_build, n_probe = int(build[0].numel()), int(probe[0].numel())
        bounds = [n_probe * i // self.n_chunks for i in range(self.n_chunks + 1)]
        if not self.segmented:
            bounds = [min(n_probe, (b + 63) // 64 * 64) for b in bounds]
        rx.next_epoch()
        self._push(0, build, build_bitmaps, None, n_build, 0, 0)
        for c in range(self.n_chunks):
            lo, hi = bounds[c], bounds[c + 1]
            self._push(1 + c, [RawCol(x.data_ptr() + lo * 8, hi - lo) for x in probe], probe_bitmaps, selected, hi - lo, 1 + c, lo, chunk=c)
        mark("pushes enqueued")
        n_out = len(self.build_types) + len(self.probe_types)
        d, keep = self._desc()
        h = C.c_void_p()
        L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
        total, result, st = 0, None, (C.c_int64 * 8)()
        out_types = (self.build_types + self.probe_types) if self.outer_is_right else (self.probe_types + self.build_types)
        try:
            if self.segmented:
                # ---- build side: the only place the host needs row counts
                rx.wait(0)
                L.check(lib.tq_compute_synchronize())        # the compute stream only: the pushes of later tables keep running
                cnt_b = rx.counts(self.rank, 0, 1)[0]
                mark("build rows arrived (host read)")
                for g in range(w):
                    if cnt_b[g]:
                        cols = [RawCol(rx.region_ptr(self.rank, 0, g, c), cnt_b[g]) for c in range(len(self.build_types))]
                        L.check(lib.tq_join_put_build(h, _tq_cols(L, cols, cnt_b[g]), L.TQ_MEM_DEVICE))
            else:
                rows = self._gather(rx, self.rank, 0, self.g_build, self.bmask)
                if rows:
                    L.check(lib.tq_join_put_build(h, self.g_build[0], L.TQ_MEM_DEVICE))
                mark("build rows arrived (gathered)")
            L.check(lib.tq_join_finalize_build(h))
            mark("build done")
            out = (L.TQColumn * n_out)()
            n, eof = C.c_int64(0), C.c_int32(0)
            chunks = []

            def drain(final):
                nonlocal total
                while True:
                    L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
                    if n.value == 0:
                        return
                    total += n.value
                    if keep_result:
                        from .chunk import device_to_host
                        if self.segmented:
                            chunks.append([device_to_host(1, out[c].data, None, n.value).values for c in range(n_out)])
                        else:
                            chunks.append([device_to_host(out_types[c], out[c].data, out[c].null_bitmap, n.value) for c in range(n_out)])
                    if not final:
                        return
            for c in range(self.n_chunks):
                if self.segmented:
                    rx.wait(1 + c)                                   # device-side: chunk c has landed from every source
                    L.check(lib.tq_join_put_probe_segments(h, w, rx.region_table(self.rank, 1 + c), rx.count_ptrs(self.rank, 1 + c), rx.cap[1 + c]))
                    mark(f"chunk {c} enqueued")
                    if c >= 1:
                        drain(False)                                 # hand back the batch before last (keeps two result sets alive, not n_chunks)
                        mark(f"chunk {c - 1} drained")
                    continue
                # gather path: a put borrows its columns until its batch is finished, so the chunk is drained before the
                # next one reuses the gather buffers
                if self._gather(rx, self.rank, 1 + c, self.g_probe, self.pmask):
                    L.check(lib.tq_join_put_probe(h, self.g_probe[0], None, L.TQ_MEM_DEVICE))
                if self.outer:
                    m = self._gather(self.misses, 0, c, self.g_miss, self.pmask)
                    if m:
                        zeros = np.zeros(m, np.uint8)
                        L.check(lib.tq_join_put_probe(h, self.g_miss[0], zeros.ctypes.data, L.TQ_MEM_DEVICE))
                drain(True)
                mark(f"chunk {c} joined")
            L.check(lib.tq_join_probe_eof(h))
            drain(True)
            mark("all drained")
            lib.tq_join_stats(h, st)
            if keep_result:
                if self.segmented:
                    result = [np.concatenate([ch[c] for ch in chunks]) if chunks else np.zeros(0, np.int64) for c in range(n_out)]
                else:
                    from .chunk import Chunk, Column
                    result = Chunk.concat([Chunk(ch) for ch in chunks], out_types).cols if chunks else [Column.empty(t, 0) for t in out_types]
        finally:
            lib.tq_join_destroy(h)
        rx.counts(self.rank)                                     # a region overflow would have dropped rows: fail loudly
        mark("overflow checks")
        dist.barrier()
        mark("barrier")
        self.last_trace = trace
        return total, list(st), result

    def _push(self, t, cols, bitmaps, selected, n, slot, row0, chunk=None):
        """push this rank's rows of table t; bitmaps / selected are taken from row row0 on"""
        bms = [None if b is None else b + row0 // 8 for b in bitmaps or []]
        if (self.bmask if t == 0 else self.pmask) and n and not any(bms):
            bms = [self._ones(n)]                      # a side declared nullable always carries the mask word: the layout is shared
        sel = None if (t == 0 or selected is None) else selected.data_ptr() + row0
        miss = (self.misses, chunk) if t > 0 and self.outer else None
        self.rx.push(t, cols, n, slot, bms, sel, miss)

    def _gather(self, layout, dst, t, target, has_mask):
        """wait (device-side) for table t of destination dst of layout from every source and copy its regions into target;
        returns the rows"""
        slots = C.c_void_p(layout.slot_ptr(dst, t, 0))
        self.L.check(self.lib.tq_region_wait(slots, layout.world, self.rx.epoch))
        n = C.c_int64(0)
        self.L.check(self.lib.tq_region_gather(layout.world, slots, layout.cap[t], layout.ncols[t] - has_mask, has_mask, layout.region_table(dst, t),
                                               target[0], target[1], C.byref(n)))
        return n.value


class VarCol:
    """a var-len device column that is just (cells pointer, offsets pointer, rows): offsets = rows + 1 int64, offsets[0] may be
    non-zero"""

    def __init__(self, data, offsets, n):
        self.data, self.offsets, self.n = data, offsets, n

    def tq(self, length=None):
        from . import _lib
        t = _lib.TQColumn()
        t.length, t.data, t.offsets = self.n if length is None else length, self.data, self.offsets
        return t


def _tq_device(L, cols, bitmaps=None):
    """(TQColumn array, rows) of device columns: objects with .tq() (DeviceColumn, DeviceVarColumn, VarCol) or (pointer,
    rows)-like ones; bitmaps, when given, replace the columns' own (a device NULL bitmap pointer or None per column)"""
    arr = (L.TQColumn * len(cols))()
    for c, x in enumerate(cols):
        if hasattr(x, "tq"):
            arr[c] = x.tq()
        else:
            arr[c].length, arr[c].data = int(x.numel()), x.data_ptr()
    n = int(arr[0].length) if len(cols) else 0
    for c in range(len(cols)):
        arr[c].length = n
    for c, b in enumerate(bitmaps or []):
        arr[c].null_bitmap = b
    return arr, n


class BroadcastJoin:
    """The multi-GPU join that replicates the build side: every rank pushes its build shard to every rank, this one
    included (tq_partition_push_broadcast), and joins its own probe shard, which never moves, against all W build shards.
    One step:

        push stream    broadcast(build shard)
        compute stream create handle + conditions | tq_region_wait (W slots) | one host read of the slots |
                       tq_join_put_build(region of source g) for g = 0..W-1 | finalize | put_probe(local shard) | eof | drain

    then one barrier (nobody may overwrite a region a peer is still building from).  The build side is the inner child, so
    the side an outer join preserves is the probe side: joining each probe shard against the whole build side is correct for
    inner, left outer and right outer joins, keyed or key-less, and every probe row's output appears on exactly one rank.  A
    key-less join puts the build regions in source order, so rank r's output is the single-GPU sequence of its probe shard
    against the rank-major concatenation of the build shards, and the ranks' outputs in rank order are the whole job's.

    Everything the single-GPU handle takes comes with it: 0..8 key columns of any 8-byte or var-len type, BYTES payloads,
    nullable columns, selected[], defaultInner and OtherConditions as comparisons or as a program.

    When to use which join: RegionJoin (the hash shuffle) moves (W-1)/W of both sides over NVLink and holds about 1/W of
    each per rank, but runs one 8-byte NOT NULL-or-masked key in column 0 over at most 4 words per row with no
    OtherConditions.  BroadcastJoin moves (W-1) x the build side over NVLink and holds W x the build side per rank, and runs
    every join the single-GPU handle runs: key-less joins, multi-column and string keys, wide rows, conditions.  It suits a
    small build side (a dimension table) or a join the shuffle cannot route; a build side that does not fit one GPU does not
    fit it."""

    def __init__(self, lib, L, world, rank, n_build_max, build_types, probe_types, build_keys=(), probe_keys=(), join_type=0,
                 outer_is_right=True, byte_caps=None, build_nullable=False, probe_nullable=False, default_inner=None,
                 other_conditions=(), other_program=(), slot=0, exchange=None):
        """n_build_max: the largest build shard; byte_caps: per build column, the most cell bytes a shard of a BYTES column
        holds (None for the others) — every rank passes the same numbers, the layout is shared.  build_types / probe_types:
        TQ_TYPE_INT64 / _UINT64 / _FLOAT64 / _BYTES.  build_keys / probe_keys: 0..8 column indices each (empty: key-less).
        other_conditions / other_program: OtherConditions over the output row as HashJoinExec takes them.  exchange: a
        RegionLayout with the attributes of a RegionExchange (rank, epoch) holding BroadcastJoin.table(...) as table 0; by
        default a RegionExchange over the ranks of the process group."""
        self.lib, self.L, self.world, self.rank, self.slot = lib, L, world, rank, slot
        self.build_types, self.probe_types = list(build_types), list(probe_types)
        self.build_keys, self.probe_keys = list(build_keys), list(probe_keys)
        if len(self.build_keys) != len(self.probe_keys) or len(self.build_keys) > 8:
            raise ValueError("BroadcastJoin: build_keys and probe_keys name the same number of columns, 0..8")
        self.join_type, self.outer_is_right, self.default_inner = join_type, bool(outer_is_right), default_inner
        self.nullable, self.probe_nullable = int(bool(build_nullable)), bool(probe_nullable)
        self.other_conditions, self.other_program = list(other_conditions), list(other_program)
        self.byte_caps = [int((byte_caps or [None] * len(self.build_types))[c] or 0) for c in range(len(self.build_types))]
        self.table = BroadcastJoin.table_of(self.build_types, n_build_max, self.byte_caps, self.nullable)
        self.rx = exchange if exchange is not None else RegionExchange(lib, L, world, rank, [self.table], align_rows=1)
        self.last_phase = {}

    @staticmethod
    def table_of(build_types, n_build_max, byte_caps, nullable):
        """the broadcast's RegionLayout table (areas, cap rows, [words per area]): per column its values or offsets, a BYTES
        column's cells, then on a nullable side its bitmap words (tq_partition_push_broadcast's order), each rounded up to
        16 bytes so every area starts 16-byte aligned"""
        from . import _lib
        cap = _round_up(max(int(n_build_max), 1), 4096)
        words = []
        for t, bc in zip(build_types, byte_caps):
            bytes_col = t == _lib.TQ_TYPE_BYTES
            words.append(_round_up(cap + (1 if bytes_col else 0), 2))
            if bytes_col:
                words.append(_round_up(max(int(bc or 0), 1), 16) // 8)
            if nullable:
                words.append(_round_up((cap + 63) // 64, 2))
        return (len(words), cap, words)

    def close(self):
        self.rx.close()

    def _areas(self, g, rows):
        """source g's build region on this rank as tq_column chunk of `rows` rows"""
        rx, L = self.rx, self.L
        arr = (L.TQColumn * len(self.build_types))()
        a = 0
        for c, t in enumerate(self.build_types):
            arr[c].length = rows
            if t == L.TQ_TYPE_BYTES:
                arr[c].offsets = rx.region_ptr(rx.rank, 0, g, a)
                arr[c].data = rx.region_ptr(rx.rank, 0, g, a + 1)
                a += 2
            else:
                arr[c].data = rx.region_ptr(rx.rank, 0, g, a)
                a += 1
            if self.nullable:
                arr[c].null_bitmap = rx.region_ptr(rx.rank, 0, g, a)
                a += 1
        return arr

    def push(self, build, build_bitmaps=None):
        """enqueue the broadcast of this rank's build shard (push stream) for the exchange's current epoch"""
        L, rx = self.L, self.rx
        arr, n = _tq_device(L, build, build_bitmaps)
        if build_bitmaps and not self.nullable:
            raise ValueError("BroadcastJoin: NULL bitmaps on the build side need build_nullable")
        types = (C.c_int32 * len(self.build_types))(*self.build_types)
        caps = (C.c_int64 * len(self.byte_caps))(*self.byte_caps)
        dest, cnts = rx.push_tables(0, rx.rank)
        L.check(self.lib.tq_partition_push_broadcast(len(self.build_types), arr, types, self.nullable, n, self.world, dest, cnts, rx.cap[0], caps,
                                                     self.slot, rx.epoch))

    def _create(self):
        L, lib = self.L, self.lib
        tb = (C.c_int32 * len(self.build_types))(*self.build_types)
        tp = (C.c_int32 * len(self.probe_types))(*self.probe_types)
        nk = len(self.build_keys)
        bk, pk = (C.c_int32 * max(nk, 1))(*self.build_keys), (C.c_int32 * max(nk, 1))(*self.probe_keys)
        d = L.TQJoinDesc(self.join_type, 1 if self.outer_is_right else 0, len(tb), tb, len(tp), tp, nk, bk if nk else None, pk if nk else None, 0, 0)
        keep = [tb, tp, bk, pk]
        if self.default_inner is not None:
            dt = {L.TQ_TYPE_INT64: np.int64, L.TQ_TYPE_UINT64: np.uint64, L.TQ_TYPE_FLOAT64: np.float64}
            keep += [(C.c_uint64 * len(tb))(*[0 if v is None else int(np.array([v], dtype=dt[t]).view(np.uint64)[0])
                                              for v, t in zip(self.default_inner, self.build_types)]),
                     (C.c_uint8 * len(tb))(*[0 if v is None else 1 for v in self.default_inner])]
            d.default_inner_bits, d.default_inner_not_null = keep[-2], keep[-1]
        h = C.c_void_p()
        L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
        try:
            if self.other_conditions:
                arr = (L.TQJoinCond * len(self.other_conditions))()
                for i, c in enumerate(self.other_conditions):
                    if c[2] is None:
                        np_t = {L.TQ_TYPE_INT64: np.int64, L.TQ_TYPE_UINT64: np.uint64, L.TQ_TYPE_FLOAT64: np.float64}[c[3]]
                        arr[i] = L.TQJoinCond(c[0], c[1], -1, c[3], int(np.array([c[4]], dtype=np_t).view(np.uint64)[0]))
                    else:
                        arr[i] = L.TQJoinCond(c[0], c[1], c[2], 0, 0)
                L.check(lib.tq_join_set_other_conditions(h, len(arr), arr))
            if self.other_program:
                from .expression import JoinProgram
                JoinProgram(self.other_program).set_on(lib.tq_join_set_other_program, h)
        except Exception:
            lib.tq_join_destroy(h)
            raise
        return h

    def join(self, probe, probe_bitmaps=None, selected=None, keep_result=False):
        """this rank's half of a step after every rank's push was enqueued: wait for the W build regions, build, probe the
        local shard, drain.  Returns (rows, stats, result); result (keep_result) = host Columns of the output"""
        lib, L, rx, w = self.lib, self.L, self.rx, self.world
        if probe_bitmaps and not self.probe_nullable:
            raise ValueError("BroadcastJoin: NULL bitmaps on the probe side need probe_nullable")
        phase, t0 = {}, time.perf_counter()

        def mark(name):
            nonlocal t0
            t1 = time.perf_counter()
            phase[name] = (t1 - t0) * 1e3
            t0 = t1
        out_types = (self.build_types + self.probe_types) if self.outer_is_right else (self.probe_types + self.build_types)
        h = self._create()
        total, chunks, st = 0, [], (C.c_int64 * 8)()
        try:
            rx.wait(0)
            cnt = rx.counts(rx.rank, 0, 1)[0]     # one host read (put_build takes host lengths); ~0 = an overflowed push: raises
            for g in range(w):
                if cnt[g]:
                    L.check(lib.tq_join_put_build(h, self._areas(g, cnt[g]), L.TQ_MEM_DEVICE))
            L.check(lib.tq_compute_synchronize())
            mark("wait + build puts")
            L.check(lib.tq_join_finalize_build(h))
            L.check(lib.tq_compute_synchronize())
            mark("finalize")
            arr, n = _tq_device(L, probe, probe_bitmaps)
            sel = None if selected is None else np.ascontiguousarray(selected, np.uint8)
            if n:
                L.check(lib.tq_join_put_probe(h, arr, None if sel is None else sel.ctypes.data, L.TQ_MEM_DEVICE))
            L.check(lib.tq_join_probe_eof(h))
            out = (L.TQColumn * len(out_types))()
            rows, eof = C.c_int64(0), C.c_int32(0)
            while True:
                L.check(lib.tq_join_next_device(h, out, C.byref(rows), C.byref(eof)))
                if rows.value == 0:
                    break
                total += rows.value
                if keep_result:
                    from .chunk import device_to_host, device_var_to_host
                    chunks.append([device_var_to_host(out[c].data, out[c].offsets, out[c].null_bitmap, rows.value) if t == L.TQ_TYPE_BYTES
                                   else device_to_host(t, out[c].data, out[c].null_bitmap, rows.value) for c, t in enumerate(out_types)])
            L.check(lib.tq_compute_synchronize())
            mark("probe + drain")
            lib.tq_join_stats(h, st)
        finally:
            lib.tq_join_destroy(h)
        result = None
        if keep_result:
            from .chunk import Chunk, Column, VarColumn
            result = (Chunk.concat([Chunk(ch) for ch in chunks], out_types).cols if chunks
                      else [(VarColumn if t == L.TQ_TYPE_BYTES else Column).empty(t, 0) for t in out_types])
        self.last_phase = phase
        return total, list(st), result

    def step_cols(self, build, probe, build_bitmaps=None, probe_bitmaps=None, selected=None, keep_result=False):
        """build / probe: this rank's shard of every column (device columns: (pointer, rows)-like objects, or VarCol /
        DeviceVarColumn for BYTES).  *_bitmaps: a device NULL bitmap pointer (or None) per column, on a side declared
        nullable.  selected: HOST bytes or bools, one per probe row (the outer-side filter), or None.  Returns (rows, stats,
        result) as RegionJoin.step_cols, result as host Columns."""
        self.rx.next_epoch()
        self.push(build, build_bitmaps)
        res = self.join(probe, probe_bitmaps, selected, keep_result)
        self.L.check(self.lib.tq_partition_push_sync(self.slot))   # the push reads the caller's build shard until it is done
        dist.barrier()
        return res


def agg_drain(lib, L, h, n_funcs):
    """the finished groups of an aggregation handle after tq_agg_eof, as host Columns: tq_agg_next_device, and — when it has
    no groups — tq_agg_next, which returns the one default row of a scalar aggregate over no rows (COUNT 0, the rest NULL)"""
    from .chunk import Column, VarColumn, device_to_host, device_var_to_host
    types = []
    for i in range(n_funcs):
        t = C.c_int32(0)
        L.check(lib.tq_agg_output_type(h, i, C.byref(t)))
        types.append(t.value)
    out = (L.TQColumn * max(n_funcs, 1))()
    rows, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_agg_next_device(h, out, C.byref(rows), C.byref(eof)))
    if rows.value:
        return [device_var_to_host(out[i].data, out[i].offsets, out[i].null_bitmap, rows.value) if types[i] == L.TQ_TYPE_BYTES
                else device_to_host(types[i], out[i].data, out[i].null_bitmap, rows.value) for i in range(n_funcs)]
    data = [np.zeros(1, np.uint64) for _ in range(n_funcs)]
    bms = [np.zeros(8, np.uint8) for _ in range(n_funcs)]
    offs = [np.zeros(2, np.int64) for _ in range(n_funcs)]
    for i in range(n_funcs):
        out[i].data, out[i].null_bitmap, out[i].offsets = data[i].ctypes.data, bms[i].ctypes.data, None
        if types[i] == L.TQ_TYPE_BYTES:
            out[i].offsets = offs[i].ctypes.data
    L.check(lib.tq_agg_next(h, 1, out, C.byref(rows), C.byref(eof)))
    if rows.value == 0:
        return [(VarColumn if t == L.TQ_TYPE_BYTES else Column).empty(t, 0) for t in types]
    return [VarColumn(t, [None if not bms[i][0] & 1 else b""]) if t == L.TQ_TYPE_BYTES else
            Column(t, data[i].view(np.float64 if t == L.TQ_TYPE_FLOAT64 else (np.uint64 if t == L.TQ_TYPE_UINT64 else np.int64)),
                   np.array([bool(bms[i][0] & 1)])) for i, t in enumerate(types)]


def partial_var_cols(types, group_by, funcs):
    """the var-len (string) partial columns of a GROUP BY, as tq_agg_push_partial_var sends them: [(partial column, input
    column)] for every GROUP BY item on a BYTES column and every MAX / MIN / FIRSTROW over a BYTES argument, in partial-column
    order (the GROUP BY items, then one column per function, two for AVG)"""
    from . import _lib
    is_bytes = [(t & 0xFF) == _lib.TQ_TYPE_BYTES for t in types]
    out, c = [], 0
    for g in group_by:
        if is_bytes[g]:
            out.append((c, g))
        c += 1
    for f, a in funcs:
        if f in (3, 4, 5) and a >= 0 and is_bytes[a]:         # TQ_AGG_MAX, TQ_AGG_MIN, TQ_AGG_FIRSTROW
            out.append((c, a))
        c += 2 if f == 2 else 1                              # TQ_AGG_AVG: (count, sum)
    return out


class RegionAgg:
    """The multi-GPU GROUP BY over a RegionExchange of one table: w + 1 wire columns (w = tq_agg_partial_width: the partial
    row, then its NULL mask word), then one byte area per var-len (string) partial column.  One step:

        this rank      Partial1 handle <- tq_agg_put(shard) -> eof -> tq_agg_push_partial_var    (push stream)
        compute stream tq_region_wait -> Final handle <- tq_agg_merge_regions_var -> eof -> next_device

    A partial group travels to the rank its group names (tq_agg_push_partial_var: with one NOT NULL 8-byte item the rank the
    join sends that key to; a string item by the content hash of its bytes), so every group is finished on exactly one rank; a
    scalar aggregate is finished on rank 0 only, which returns its one row even when every shard is empty.  A string partial
    column travels as offsets plus its cells, which the receiver encodes into its own dictionary.  Without string columns the
    wire format is tq_agg_push_partial's.  Host synchronisation per step: the export's group count, the merge's slot read (and
    one byte-total read per string column and region), the result drain and ONE barrier at the end (nobody may push into a
    region a peer is still merging)."""

    def __init__(self, lib, L, world, rank, types, group_by, funcs, max_groups_per_rank, slack=1.25, est_groups=0, slot=0, byte_caps=None,
                 exchange=None):
        """types: TQ_TYPE_* per input column (| TQ_TYPE_NOT_NULL where declared so); group_by: input column indices;
        funcs: [(TQ_AGG_*, arg_col)].  max_groups_per_rank: the most groups one rank's shard holds; byte_caps: per input
        column, for a BYTES column the most cell bytes one rank's partial rows hold in one partial column of it (at most the
        bytes of the shard's column), None for the others.  Every rank passes the same numbers: the layout is shared.
        exchange: a RegionLayout with the attributes of a RegionExchange (rank, epoch, wait, next_epoch) holding
        RegionAgg.table_of(...) as table 0; by default a RegionExchange over the ranks of the process group."""
        self.lib, self.L, self.world, self.rank, self.slot = lib, L, world, rank, slot
        self.types, self.group_by, self.funcs, self.est_groups = list(types), list(group_by), list(funcs), est_groups
        h, keep = self._create()
        try:
            width = C.c_int32(0)
            L.check(lib.tq_agg_partial_width(h, C.byref(width)))
        finally:
            lib.tq_agg_destroy(h)
        self.width = width.value
        if self.width + 1 > 64:
            raise ValueError(f"RegionAgg: {self.width} partial columns and the mask word exceed 64 words per row")
        self.var_cols = partial_var_cols(self.types, self.group_by, self.funcs)
        self.table, self.byte_cap = RegionAgg.table_of(world, self.width, self.var_cols, bool(group_by), max_groups_per_rank, byte_caps, slack)
        self.rx = exchange if exchange is not None else RegionExchange(lib, L, world, rank, [self.table])
        self._hp = None
        self.last_phase = {}

    @staticmethod
    def table_of(world, width, var_cols, grouped, max_groups_per_rank, byte_caps=None, slack=1.25):
        """(the RegionLayout table, the byte cap of every var-len partial column): width + 1 word areas of cap rows (a var-len
        column's area is cap + 1 offsets, rounded up to 16 bytes), then one byte area per var-len column.  Rows and bytes take
        the same slack: a group lands on one rank by its hash, so +25 % (and a fixed margin) covers the imbalance between
        (source, destination) pairs.  Without var-len columns it is (width + 1, cap)."""
        cap = _round_up(1 if not grouped else int(max_groups_per_rank / world * slack) + (1 << 14), 4096)
        if not var_cols:
            return (width + 1, cap), []
        byte_cap = []
        for _, src in var_cols:
            most = byte_caps[src] if byte_caps and src < len(byte_caps) else None
            if most is None:
                raise ValueError(f"RegionAgg: input column {src} is a string column and needs byte_caps[{src}]")
            b = _round_up(int(int(most) / world * slack) + (1 << 14), 16)
            if b >= 1 << 32:
                raise ValueError(f"RegionAgg: {b} bytes per region for input column {src}: at most 2^32 - 16")
            byte_cap.append(b)
        var = {c for c, _ in var_cols}
        words = [_round_up(cap + 1, 2) if c in var else cap for c in range(width)] + [cap] + [b // 8 for b in byte_cap]
        return (len(words), cap, words), byte_cap

    def _create(self):
        L = self.L
        it = (C.c_int32 * len(self.types))(*self.types)
        gb = (C.c_int32 * max(len(self.group_by), 1))(*self.group_by)
        fa = (L.TQAggFunc * max(len(self.funcs), 1))(*[L.TQAggFunc(f, a) for f, a in self.funcs])
        d = L.TQAggDesc(len(self.types), it, len(self.group_by), gb, len(self.funcs), fa, self.est_groups)
        h = C.c_void_p()
        L.check(self.lib.tq_agg_create(C.byref(d), C.byref(h)))
        return h, (it, gb, fa)

    def close(self):
        self.rx.close()

    def merge_table(self, dst):
        """destination dst's regions as tq_agg_merge_regions_var takes them: regions[g * (w + 1) + c], a var-len column with
        .offsets = its word area and .data = its byte area"""
        rx, nw = self.rx, self.width + 1
        regs = (self.L.TQColumn * (self.world * nw))()
        for g in range(self.world):
            for c in range(nw):
                regs[g * nw + c].length, regs[g * nw + c].data = rx.cap[0], rx.region_ptr(dst, 0, g, c)
            for v, (c, _) in enumerate(self.var_cols):
                regs[g * nw + c].offsets = regs[g * nw + c].data
                regs[g * nw + c].data = rx.region_ptr(dst, 0, g, nw + v)
        return regs

    def push(self, cols, bitmaps=None):
        """this rank's half of a step before the merge: aggregate the shard into a Partial1 handle and enqueue its push (push
        stream) for the exchange's current epoch.  cols: this rank's shard of every input column ((device pointer,
        rows)-like objects, or VarCol / DeviceVarColumn for BYTES); bitmaps: a device NULL bitmap pointer (or None) per
        column.  The handle is read until tq_partition_push_sync(slot)."""
        lib, L, rx = self.lib, self.L, self.rx
        arr, n = _tq_device(L, cols, bitmaps)
        hp, _ = self._create()
        self._hp = hp
        if n:
            L.check(lib.tq_agg_put(hp, arr, L.TQ_MEM_DEVICE))
        L.check(lib.tq_agg_eof(hp))
        dest, cnts = rx.push_tables(0, self.rank)
        caps = (C.c_int64 * max(len(self.byte_cap), 1))(*self.byte_cap)
        L.check(lib.tq_agg_push_partial_var(hp, self.world, dest, cnts, rx.cap[0], caps, self.slot, rx.epoch))

    def finish(self, keep_result=False):
        """this rank's half after every rank's push was enqueued: wait, merge, finish.  Returns (groups finished on this rank,
        result): result (keep_result) = host Columns of the function outputs, None otherwise.  A region past its row or byte
        cap is TQ_ERR_OOM (RuntimeError)."""
        lib, L, rx = self.lib, self.L, self.rx
        hf, keep_f = self._create()
        try:
            rx.wait(0)
            L.check(lib.tq_agg_merge_regions_var(hf, self.world, C.c_void_p(rx.slot_ptr(self.rank, 0, 0)), rx.cap[0], self.merge_table(self.rank)))
            L.check(lib.tq_agg_eof(hf))
            L.check(lib.tq_partition_push_sync(self.slot))     # the push reads the Partial1 handle's rows until it is done
            res, groups = None, 0
            if keep_result and (self.group_by or self.rank == 0):
                res = agg_drain(lib, L, hf, len(self.funcs))
                groups = res[0].length if res else 0
            elif self.group_by or self.rank == 0:
                out = (L.TQColumn * max(len(self.funcs), 1))()
                rows, eof = C.c_int64(0), C.c_int32(0)
                L.check(lib.tq_agg_next_device(hf, out, C.byref(rows), C.byref(eof)))   # the groups stay in HBM
                if rows.value or self.group_by:
                    groups = rows.value
                else:                                        # a scalar aggregate over no rows: the default row, unless all FIRSTROW
                    groups = int(any(f != 5 for f, _ in self.funcs))
        finally:
            if self._hp is not None:
                lib.tq_partition_push_sync(self.slot)
                lib.tq_agg_destroy(self._hp)
                self._hp = None
            lib.tq_agg_destroy(hf)
        return groups, res

    def step(self, cols, bitmaps=None, keep_result=False):
        """one step on this rank: push, wait, merge, finish, then one barrier.  cols / bitmaps as push().  Returns (groups
        finished on this rank, result) as finish().  A step that fails on any rank raises on this one too when the failure
        reaches it (a push that fails after its checks makes every merge refuse the step); the barrier is passed either way, so
        the ranks leave a failed step together and the next step runs as usual."""
        self.rx.next_epoch()
        try:
            self.push(cols, bitmaps)
            res = self.finish(keep_result)
        finally:
            if self._hp is not None:
                self.lib.tq_partition_push_sync(self.slot)
                self.lib.tq_agg_destroy(self._hp)
                self._hp = None
            dist.barrier()
        return res


class RegionSort:
    """The multi-GPU ORDER BY and ORDER BY ... LIMIT over a RegionExchange of two tables: 0 = the splitter sample (the
    broadcast's wire format: the ByItem columns, then the tie word), 1 = the rows (the GROUP BY push's wire format: one word
    area per column, a BYTES column's being its offsets, the mask word, then one byte area per BYTES column).  Rank r holds
    shard r; the global order is tq_sort of the shards concatenated in rank order (equal keys keep that order).

    ORDER BY (limit_count < 0): rank d ends up with the d-th contiguous slice of the global order.

        push stream    tq_partition_push_sample (min(n, n_samples) rows + tie words to every rank)
        compute stream tq_region_wait | tq_sort of the W sample regions, by the ByItems then the tie word | splitters at
                       rows floor(k m / W), k = 1 .. W - 1, of the m sample rows (the same on every rank, no host comparator)
        push stream    tq_partition_push_ranges (row -> the splitters at or below (its keys, its tie word))
        compute stream tq_region_wait | tq_sort_put_regions (sources in rank order) | eof | drain

    The tie word (src_rank << 32) | row is the last, ascending ByItem of the routing only: it makes the routing order total
    and equal to the global order, so a run of equal keys is split between ranks wherever the splitters fall (a column of one
    value spreads evenly), and the rows a rank receives from the sources, put in rank order and sorted stably, are its slice.

    ORDER BY ... LIMIT (limit_count >= 0): each rank sorts its shard with limit (0, limit_offset + limit_count) and pushes
    that result to rank 0 (tq_partition_push_ranges, one destination); rank 0 sorts the W regions with the real limit and
    holds rows [limit_offset, limit_offset + limit_count) of the global order, every other rank none.

    Sizing: every (source, destination) region holds a whole shard (n_max rows) and each byte area a shard's cells
    (byte_caps), so no push overflows on rows: the splitters decide only how evenly the work spreads.  The price is W x the
    largest shard held per rank for the rows (the cost BroadcastJoin pays for its build side), plus a sample table of W x
    min(n_max, n_samples) rows whose byte areas also take byte_caps (the sampled rows are distinct, so their cells never
    exceed the shard's)."""

    def __init__(self, lib, L, world, rank, types, by_cols, by_desc, n_max, byte_caps=None, nullable=False, limit_offset=0, limit_count=-1,
                 n_samples=1024, slot=0, exchange=None, seed=0x5EED5EED):
        """types: TQ_TYPE_INT64 / _UINT64 / _FLOAT64 / _BYTES per column; by_cols / by_desc: the 0..8 ByItems; n_max: the
        largest shard; byte_caps: per column, for a BYTES column the most cell bytes one shard holds (None for the others);
        nullable: the columns may carry NULL bitmaps (the sample then carries bitmap words).  Every rank passes the same
        numbers: the layout is shared.  exchange: a RegionLayout with the attributes of a RegionExchange (rank, epoch, wait,
        next_epoch) holding RegionSort.table_of(...) as tables 0 and 1; by default a RegionExchange over the process group."""
        self.lib, self.L, self.world, self.rank, self.slot = lib, L, world, rank, slot
        self.types, self.by_cols, self.by_desc = [t & 0xFF for t in types], list(by_cols), [int(bool(d)) for d in by_desc]
        if len(self.by_cols) != len(self.by_desc) or len(self.by_cols) > 8:
            raise ValueError("RegionSort: by_cols and by_desc name the same 0..8 ByItems")
        self.nullable = int(bool(nullable))
        self.limit_offset, self.limit_count = int(limit_offset), int(limit_count)
        self.n_samples, self.seed = int(n_samples), int(seed)
        self.byte_caps = [int((byte_caps or [None] * len(self.types))[c] or 0) for c in range(len(self.types))]
        self.tables = RegionSort.table_of(self.types, self.by_cols, n_max, self.byte_caps, self.nullable, self.n_samples)
        self.rx = exchange if exchange is not None else RegionExchange(lib, L, world, rank, self.tables, align_rows=1)
        self._handles = []   # sort handles whose lent results a push may still read

    @staticmethod
    def table_of(types, by_cols, n_max, byte_caps, nullable, n_samples=1024):
        """[the sample table, the rows table] as RegionLayout tables.  The sample is BroadcastJoin.table_of over the ByItem
        columns and the tie word (UINT64) at min(n_max, n_samples) rows; the rows table has n_max rows per region: per column
        n_max words (a BYTES column: n_max + 1 offsets), the mask word, then a byte area of byte_caps[c] bytes per BYTES
        column, every area rounded up to 16 bytes."""
        from . import _lib
        types = [t & 0xFF for t in types]
        is_b = [t == _lib.TQ_TYPE_BYTES for t in types]
        caps = [int((byte_caps or [None] * len(types))[c] or 0) for c in range(len(types))]
        for c in range(len(types)):
            if is_b[c] and not 1 <= caps[c] < (1 << 32) - 16:
                raise ValueError(f"RegionSort: BYTES column {c} needs 1 <= byte_caps[{c}] < 2^32 - 16")
        sample = BroadcastJoin.table_of([types[b] for b in by_cols] + [_lib.TQ_TYPE_UINT64], min(max(int(n_max), 1), int(n_samples)),
                                        [caps[b] for b in by_cols] + [None], nullable)
        cap = _round_up(max(int(n_max), 1), 2)
        words = [_round_up(cap + 1, 2) if b else cap for b in is_b] + [cap] + [_round_up(caps[c], 16) // 8 for c in range(len(types)) if is_b[c]]
        return [sample, (len(words), cap, words)]

    def close(self):
        self.rx.close()

    def _sample_areas(self, g, rows):
        """source g's sample region on this rank as a tq_column chunk of `rows` rows (ByItem columns, then the tie word)"""
        rx, L = self.rx, self.L
        st = [self.types[b] for b in self.by_cols] + [L.TQ_TYPE_UINT64]
        arr = (L.TQColumn * len(st))()
        a = 0
        for c, t in enumerate(st):
            arr[c].length = rows
            if t == L.TQ_TYPE_BYTES:
                arr[c].offsets, arr[c].data = rx.region_ptr(rx.rank, 0, g, a), rx.region_ptr(rx.rank, 0, g, a + 1)
                a += 2
            else:
                arr[c].data = rx.region_ptr(rx.rank, 0, g, a)
                a += 1
            if self.nullable:
                arr[c].null_bitmap = rx.region_ptr(rx.rank, 0, g, a)
                a += 1
        return arr

    def _published(self, t):
        """one host read of this rank's slots of table t after its wait: a slot that does not carry this epoch (a peer that
        never pushed) raises RuntimeError.  Returns the slots' rows words"""
        rx = self.rx
        self.L.check(self.lib.tq_compute_synchronize())
        raw = rx.read_slots(rx.rank, t, 1)[0]
        late = [g for g in range(self.world) if int(raw[g, 1]) != rx.epoch]
        if late:
            raise RuntimeError(f"RegionSort: sources {late} did not publish table {t} for epoch {rx.epoch}")
        return [int(x) for x in raw[:, 0]]

    def _sort(self, n_cols, types, by_cols, by_desc, limit_offset, limit_count):
        L = self.L
        tt = (C.c_int32 * n_cols)(*types)
        bc, bd = (C.c_int32 * max(len(by_cols), 1))(*by_cols), (C.c_int32 * max(len(by_desc), 1))(*by_desc)
        d = L.TQSortDesc(n_cols, tt, len(by_cols), bc, bd, limit_offset, limit_count)
        h = C.c_void_p()
        L.check(self.lib.tq_sort_create(C.byref(d), C.byref(h)))
        self._handles.append(h)
        return h

    def _lend(self, h, n_cols):
        out = (self.L.TQColumn * n_cols)()
        rows, eof = C.c_int64(0), C.c_int32(0)
        self.L.check(self.lib.tq_sort_next_device(h, out, C.byref(rows), C.byref(eof)))
        return out, rows.value

    def push_sample(self, cols, bitmaps=None):
        """ORDER BY: enqueue the push of this rank's splitter sample (push stream) for the exchange's current epoch.  cols:
        this rank's shard of every column ((device pointer, rows)-like objects, or VarCol / DeviceVarColumn for BYTES);
        bitmaps: a device NULL bitmap pointer (or None) per column"""
        L, rx = self.L, self.rx
        arr, n = _tq_device(L, cols, bitmaps)
        nb = len(self.by_cols)
        types, by = (C.c_int32 * len(self.types))(*self.types), (C.c_int32 * max(nb, 1))(*self.by_cols)
        caps = (C.c_int64 * len(self.byte_caps))(*self.byte_caps)
        dest, cnts = rx.push_tables(0, self.rank)
        L.check(self.lib.tq_partition_push_sample(len(self.types), arr, types, n, nb, by, self.nullable, self.rank, self.n_samples, self.seed,
                                                  self.world, dest, cnts, rx.cap[0], caps, self.slot, rx.epoch))

    def push_rows(self, cols, bitmaps=None):
        """enqueue the push of this rank's rows (push stream): ORDER BY after every rank's push_sample (this waits for the
        samples and sorts them), TopN on its own.  The shard (and the handles lent to the push) are read until
        tq_partition_push_sync(slot)."""
        L, lib, rx, w = self.L, self.lib, self.rx, self.world
        arr, n = _tq_device(L, cols, bitmaps)
        nc, nb = len(self.types), len(self.by_cols)
        types, by = (C.c_int32 * nc)(*self.types), (C.c_int32 * max(nb, 1))(*self.by_cols)
        desc = (C.c_int32 * max(nb, 1))(*self.by_desc)
        caps = (C.c_int64 * nc)(*self.byte_caps)
        split, m, pos = None, 0, None
        if self.limit_count >= 0:                 # TopN: this shard's first limit_offset + limit_count rows, to rank 0
            h = self._sort(nc, self.types, self.by_cols, self.by_desc, 0, self.limit_offset + self.limit_count)
            if n:
                L.check(lib.tq_sort_put(h, arr, L.TQ_MEM_DEVICE))
            L.check(lib.tq_sort_eof(h))
            arr, n = self._lend(h, nc)
            if n == 0:
                arr = _tq_device(L, cols, bitmaps)[0]
            dest, cnts = rx.push_tables(1, self.rank)
            n_parts = 1
        else:                                     # ORDER BY: the splitters from the W samples, then every row to its rank
            rx.wait(0)
            self._published(0)
            cnt = rx.counts(rx.rank, 0, 1)[0]          # a sample push that failed or overflowed raises here, on every rank
            st = [self.types[b] for b in self.by_cols] + [L.TQ_TYPE_UINT64]
            h = self._sort(nb + 1, st, list(range(nb + 1)), self.by_desc + [0], 0, -1)
            for g in range(w):
                if cnt[g]:
                    L.check(lib.tq_sort_put(h, self._sample_areas(g, cnt[g]), L.TQ_MEM_DEVICE))
            L.check(lib.tq_sort_eof(h))
            split, m = self._lend(h, nb + 1)
            pos = (C.c_int64 * max(w - 1, 1))(*[k * m // w for k in range(1, w)])
            dest, cnts = rx.push_tables(1, self.rank)
            n_parts = w
        L.check(lib.tq_partition_push_ranges(nc, arr, types, n, nb, by, desc, self.rank, n_parts, split, m, pos, dest, cnts, rx.cap[1], caps,
                                             self.slot, rx.epoch))

    def finish(self, keep_result=False):
        """this rank's half after every rank's push_rows: wait, put the regions in rank order, sort, drain.  Returns (rows on
        this rank, result): result (keep_result) = host Columns of this rank's rows in order, None otherwise.  A region past
        its byte cap, or a source whose push failed, raises (TQError) on every rank."""
        lib, L, rx, w = self.lib, self.L, self.rx, self.world
        nc = len(self.types)
        try:
            if self.limit_count >= 0 and self.rank != 0:
                return 0, None
            rx.wait(1)
            self._published(1)                         # a failed or overflowed source: tq_sort_put_regions refuses the step
            h = self._sort(nc, self.types, self.by_cols, self.by_desc, self.limit_offset if self.limit_count >= 0 else 0, self.limit_count)
            regs = (L.TQColumn * (w * (nc + 1)))()
            for g in range(w):
                v = 0
                for c in range(nc + 1):
                    k = g * (nc + 1) + c
                    regs[k].length, regs[k].data = rx.cap[1], rx.region_ptr(rx.rank, 1, g, c)
                    if c < nc and self.types[c] == L.TQ_TYPE_BYTES:
                        regs[k].offsets, regs[k].data = regs[k].data, rx.region_ptr(rx.rank, 1, g, nc + 1 + v)
                        v += 1
            L.check(lib.tq_sort_put_regions(h, w, C.c_void_p(rx.slot_ptr(rx.rank, 1, 0)), rx.cap[1], regs))
            L.check(lib.tq_sort_eof(h))
            out, rows = self._lend(h, nc)
            res = None
            if keep_result:
                from .chunk import Column, VarColumn, device_to_host, device_var_to_host
                res = ([device_var_to_host(out[c].data, out[c].offsets, out[c].null_bitmap, rows) if t == L.TQ_TYPE_BYTES
                        else device_to_host(t, out[c].data, out[c].null_bitmap, rows) for c, t in enumerate(self.types)] if rows
                       else [(VarColumn if t == L.TQ_TYPE_BYTES else Column).empty(t, 0) for t in self.types])
            return rows, res
        finally:
            self.release()

    def release(self):
        """wait for this rank's pushes and free what they read"""
        self.lib.tq_partition_push_sync(self.slot)
        for h in self._handles:
            self.lib.tq_sort_destroy(h)
        self._handles = []

    def step(self, cols, bitmaps=None, keep_result=False):
        """one step on this rank: (sample push, splitters,) row push, wait, put, sort, drain, then one all-gather of the W row
        counts and one barrier.  Returns (rows on this rank, global position of its first row, result) — for TopN rank 0's
        position is limit_offset.  A step that fails on any rank fails on every rank (a push that fails after its checks
        makes every receiver refuse the step); the barrier is passed either way, so the ranks leave a failed step together
        and the next step reuses the regions."""
        self.rx.next_epoch()
        rows, res, err = 0, None, None
        try:
            if self.limit_count < 0:
                self.push_sample(cols, bitmaps)
            self.push_rows(cols, bitmaps)
            rows, res = self.finish(keep_result)
        except Exception as e:
            err = e
        finally:
            self.release()
            counts = [None] * self.world
            dist.all_gather_object(counts, None if err is not None else rows)
            dist.barrier()
        if err is not None:
            raise err
        failed = [g for g, c in enumerate(counts) if c is None]
        if failed:
            raise RuntimeError(f"RegionSort: the step failed on ranks {failed}")
        return rows, (self.limit_offset if self.limit_count >= 0 else 0) + sum(counts[:self.rank]), res


def gen_dist_tables(rank, world, n_b, n_p):
    """this rank's shard of the C5 tables: B.k = the keys k with k % world == rank (shuffled), B.v = 7k + 1; probe row i of
    rank r has the global id g = r * n_p + i, P.v = g and P.k = mix64(g) % (n_b * world) — uniform keys, every probe row
    matches exactly once, and any rank can check any row it receives from its values alone."""
    rng = np.random.default_rng(1000 + rank)
    bk = rng.permutation(n_b).astype(np.int64) * world + rank
    gid = np.arange(n_p, dtype=np.int64) + rank * n_p
    pk = (mix64_np(gid) % np.uint64(n_b * world)).astype(np.int64)
    return bk, bk * 7 + 1, pk, gid


def verify_dist_result(cols, rank, world, n_b, n_p):
    """every row this rank produced: B.v = 7 B.k + 1, B.k = P.k, P.k = mix64(P.v) % N_b (the key that probe row really carried),
    the key belongs to this rank's hash partition, no probe row twice.  Returns (ok, rows, wrapping sum of P.v)."""
    bk, bv, pkk, pv = cols
    ok = bool(np.array_equal(bv, bk * 7 + 1) and np.array_equal(bk, pkk))
    ok = ok and bool(np.array_equal(pkk, (mix64_np(pv) % np.uint64(n_b * world)).astype(np.int64)))
    ok = ok and bool((dest_rank_np(pkk, world) == rank).all())
    ok = ok and bool(np.unique(pv).size == pv.size)
    return ok, int(pv.size), int(pv.astype(np.uint64).sum(dtype=np.uint64))


def dist_sizes(args):
    """per-GPU (build, probe) rows of the N > 1 line: C5's 1e8 x 1e9 at 8 GPUs = 1.25e7 / 1.25e8 per GPU at every N, unless
    --build-rows / --probe-rows override the per-GPU sizes"""
    default_sizes = (args.build_rows, args.probe_rows) == (10_000_000, 100_000_000)
    return (12_500_000, 125_000_000) if default_sizes else (args.build_rows, args.probe_rows)


def dist_workload_config(world, n_b, n_p, n_chunks=None):
    """the `config` of the N > 1 bench line; the reference arm (--impl reference --gpus N) reports the same workload"""
    N_b, N_p = n_b * world, n_p * world
    cfg = {"workload": f"C5: int64 equi-join radix-partitioned on the key over {world} GPUs; per GPU build={n_b} probe={n_p} (global {N_b} x {N_p}), "
                       "uniform keys, 100% match, output (B.k,B.v,P.k,P.v) materialised in HBM on the rank that owns the key",
           "build_rows_per_gpu": n_b, "probe_rows_per_gpu": n_p, "global_build_rows": N_b, "global_probe_rows": N_p,
           "exchange": "fused scatter + push into per-source regions of the peers' receive buffers (CUDA IPC peer stores over NVLink), device-side epoch "
                       "flags instead of host barriers; local join reads the regions as one segmented batch",
           "l2": "inputs and outputs exceed the 50 MB L2; no flush needed"}
    if n_chunks is not None:
        cfg["parallelism"] = f"key-hash partitions over {world} ranks, {n_chunks} probe chunks pipelined (push of chunk c+1 overlaps the join of chunk c)"
    return cfg


def bench_distributed_join(args, rank, world, local_rank, dist_mod, peak, peak_src):
    """bench.py N>1.  Default tables: C5 — build 1e8 / probe 1e9 at 8 GPUs, i.e. 1.25e7 / 1.25e8 rows PER GPU at every N
    (weak scaling: per-GPU work is fixed); --build-rows / --probe-rows override the per-GPU sizes."""
    import statistics

    from . import _lib as L
    lib = L.load()
    dev = torch.device("cuda", local_rank)
    n_b, n_p = dist_sizes(args)
    N_b, N_p = n_b * world, n_p * world
    bk_h, bv_h, pk_h, pv_h = gen_dist_tables(rank, world, n_b, n_p)
    bk, bv, pk, pv = (torch.from_numpy(x).to(dev) for x in (bk_h, bv_h, pk_h, pv_h))
    del bk_h, bv_h, pv_h
    torch.cuda.synchronize()
    n_chunks = max(1, int(os.environ.get("TQ_DIST_CHUNKS", "2")))   # probe chunks per step: fewer chunks, fewer exchanges
    rj = RegionJoin(lib, L, world, rank, n_b, n_p, n_chunks)

    def step(keep=False):
        return rj.step(bk, bv, pk, pv, keep_result=keep)

    for _ in range(args.warmup):
        step()
    from bench import ClockSampler
    sampler = ClockSampler(local_rank)
    sampler.start()
    torch.cuda.synchronize()
    lib.tq_device_synchronize()
    dist_mod.barrier()
    launches1 = lib.tq_kernel_launch_count()
    L.check(lib.tq_timer_start())
    t0 = time.perf_counter()
    rows_total, probe_ns, build_ns, traces = 0, [], [], []
    for _ in range(args.steps):
        rows, st, _ = step()
        traces.append(rj.last_trace)
        rows_total += rows
        probe_ns.append(st[5])
        build_ns.append(st[6])
    ms = C.c_float(0)
    L.check(lib.tq_timer_stop(C.byref(ms)))
    lib.tq_device_synchronize()
    wall_ms = (time.perf_counter() - t0) * 1e3
    dist_mod.barrier()
    clocks = sampler.stop()
    launches2 = lib.tq_kernel_launch_count()
    t = torch.tensor([ms.value, float(rows_total), wall_ms], dtype=torch.float64, device=dev)
    tmax = t.clone()
    dist_mod.all_reduce(tmax, op=dist_mod.ReduceOp.MAX)
    tsum = t.clone()
    dist_mod.all_reduce(tsum, op=dist_mod.ReduceOp.SUM)
    ms_per_step = float(tmax[0]) / args.steps
    joined_per_step = float(tsum[1]) / args.steps
    value = joined_per_step / (ms_per_step * 1e-3)
    # ---- full-size value check at this N (outside the timed region): every rank verifies every row it produced
    rows_v, _, res = step(keep=True)
    ok, n_rows, pv_sum = verify_dist_result(res, rank, world, n_b, n_p)
    del res
    v = torch.tensor([1 if ok else 0, n_rows, pv_sum % (1 << 62), pv_sum >> 62], dtype=torch.int64, device=dev)
    vmin = v.clone()
    dist_mod.all_reduce(vmin, op=dist_mod.ReduceOp.MIN)
    vsum = v.clone()
    dist_mod.all_reduce(vsum, op=dist_mod.ReduceOp.SUM)
    want_sum = (N_p * (N_p - 1) // 2) % (1 << 64)
    got_sum = ((int(vsum[3]) << 62) + int(vsum[2])) % (1 << 64)
    verified = {"ok": bool(int(vmin[0]) == 1 and int(vsum[1]) == N_p and got_sum == want_sum), "rows": int(vsum[1]), "expected_rows": N_p,
                "checks": ["per rank, every row: B.v == 7*B.k + 1, B.k == P.k, P.k == mix64(P.v) % N_build, dest_rank(P.k) == rank, P.v distinct",
                           "all ranks: row count == probe rows, sum(P.v) == N(N-1)/2 (every probe row exactly once)"]}
    # ---- the exchange north_star names, measured once for the record: partition + ONE grouped NCCL send/recv (all-to-all)
    nccl_ms = None
    lean = os.environ.get("TQ_DIST_LEAN", "0") == "1"   # quick validation runs: skip the NCCL comparison and the one-GPU baseline
    try:
        if lean:
            raise RuntimeError("skipped (TQ_DIST_LEAN=1)")
        part = gpu_partition_fn(lib, L)
        torch.cuda.synchronize()
        dist_mod.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        p_part, p_off = part([pk, pv], world)
        torch.cuda.synchronize()
        cnt = exchange_counts([p_off], world, rank, dev)[0]
        p_recv, _ = exchange(p_part, p_off, world, rank, recv_counts=cnt)   # warm-up: connection setup and buffer registration
        del p_recv
        torch.cuda.synchronize()
        dist_mod.barrier()
        e0.record()
        p_recv, _ = exchange(p_part, p_off, world, rank, recv_counts=cnt)
        e1.record()
        torch.cuda.synchronize()
        tn = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
        dist_mod.all_reduce(tn, op=dist_mod.ReduceOp.MAX)
        nccl_ms = float(tn[0])
        del p_part, p_recv
    except Exception as e:  # diagnostics only
        nccl_ms = f"unavailable: {type(e).__name__}: {e}"
    # ---- strong-scaling reference: the WHOLE job (N_b x N_p) on ONE GPU (rank 0), same kernels, no exchange
    one_gpu = None
    if os.environ.get("TQ_DIST_ONE_GPU", "1") == "1" and not lean:
        rj.close()
        rj = None
        del bk, bv, pk, pv
        torch.cuda.empty_cache()
        if rank == 0:
            try:
                one_gpu = one_gpu_reference(lib, L, dev, world, n_b, n_p)
            except Exception as e:
                one_gpu = {"error": f"{type(e).__name__}: {e}"}
        dist_mod.barrier()
    if rj is not None:
        rj.close()
    probe_s = statistics.mean(probe_ns) * 1e-9
    if rank != 0:
        return None
    push_bytes = 16.0 * n_p * (world - 1) / world
    out = {
        "metric": "joined rows/sec on 1e8-row int64 equi-join", "value": value, "unit": "joined rows/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "int64",
        "data": "synthetic",
        "config": dist_workload_config(world, n_b, n_p, n_chunks),
        "roofline": {"bound": "nvlink", "kernel": "push of this rank's probe rows (7/8 of them cross NVLink at 8 GPUs), overlapped with the local join",
                     "achieved": push_bytes / (ms_per_step * 1e-3) / 1e9, "peak": 450.0, "unit": "GB/s", "frac": push_bytes / (ms_per_step * 1e-3) / 1e9 / 450.0,
                     "traffic": None, "peak_source": "H100 SXM data sheet: NVLink 900 GB/s per GPU, 450 GB/s per direction",
                     "note": "whole-step time charged against the NVLink bytes one GPU must send; local probe pipeline of rank 0: "
                             f"{probe_s * 1e3:.3f} ms per chunk batch, build {statistics.mean(build_ns) * 1e-6:.3f} ms"},
        "e2e": {"value": value, "unit": "joined rows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0,
                "note": "multi-GPU line: shards are generated in HBM; the host-buffer e2e figure is reported on the 1-GPU line"},
        "verified": verified,
        "phase_ms_rank0": {name: round(statistics.mean(tr[i][1] for tr in traces), 3) for i, (name, _) in enumerate(traces[0])},
        "phase_note": "host-side timeline of one step on rank 0 (ms since the step began, mean over the timed steps): the points where the host thread resumes",
        "nccl_all_to_all_probe_exchange_ms": nccl_ms,
        "one_gpu_same_job": one_gpu,
        "gpu_launches": int(launches2 - launches1), "clocks": clocks, "wall_ms_per_step_max": float(tmax[2]) / args.steps,
    }
    if isinstance(one_gpu, dict) and "ms_per_step" in one_gpu:
        out["speedup_vs_one_gpu_same_job"] = one_gpu["ms_per_step"] / ms_per_step
    return out


def one_gpu_reference(lib, L, dev, world, n_b, n_p, steps=2):
    """The whole C5 job on ONE GPU: build N_b rows, probe N_p rows in `world` device batches (same generators).  This is the
    denominator of the strong-scaling figure north_star asks for (>= 4x at 8 GPUs on the 1e9-row join)."""
    N_b = n_b * world
    bk = torch.cat([torch.from_numpy(np.random.default_rng(1000 + r).permutation(n_b).astype(np.int64) * world + r).to(dev) for r in range(world)])
    bv = bk * 7 + 1
    shards = []
    for r in range(world):   # all N_p probe rows resident (16 bytes each): generated once, outside the timed region
        gid = torch.arange(n_p, dtype=torch.int64, device=dev) + r * n_p
        shards.append((_mix64_mod_torch(gid, N_b), gid))
    torch.cuda.synchronize()
    t = (C.c_int32 * 2)(1, 1)
    k = (C.c_int32 * 1)(0)
    best = None
    rows = 0
    for it in range(steps + 1):
        lib.tq_device_synchronize()
        ms = C.c_float(0)
        if it > 0:
            L.check(lib.tq_timer_start())
        d = L.TQJoinDesc(0, 1, 2, t, 2, t, 1, k, k, 0, 0)
        h = C.c_void_p()
        L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
        try:
            L.check(lib.tq_join_put_build(h, _tq_cols(L, [bk, bv], N_b), L.TQ_MEM_DEVICE))
            L.check(lib.tq_join_finalize_build(h))
            out = (L.TQColumn * 4)()
            n, eof = C.c_int64(0), C.c_int32(0)
            rows = 0
            for r in range(world):
                pk, gid = shards[r]
                L.check(lib.tq_join_put_probe(h, _tq_cols(L, [pk, gid], n_p), None, L.TQ_MEM_DEVICE))
                while True:
                    L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
                    if n.value == 0:
                        break
                    rows += n.value
                    if r < world - 1:
                        break
            L.check(lib.tq_join_probe_eof(h))
            while True:
                L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
                if n.value == 0:
                    break
                rows += n.value
        finally:
            lib.tq_join_destroy(h)
        if it > 0:
            L.check(lib.tq_timer_stop(C.byref(ms)))
            best = ms.value if best is None else min(best, ms.value)
    return {"ms_per_step": best, "rows": int(rows), "value": rows / (best * 1e-3), "build_rows": N_b, "probe_rows": n_p * world,
            "note": "one GPU, all inputs resident in HBM before the timed region, probe fed in device batches of one shard each; best of the timed repetitions"}


def _mix64_mod_torch(gid, mod):
    """mix64(g) % mod on the device with int64 tensors (wrapping multiply; logical shifts emulated)"""
    def shr(x, s):
        return (x >> s) & ((1 << (64 - s)) - 1)
    k = gid.clone()
    k ^= shr(k, 33)
    k *= -49064778989728563          # 0xff51afd7ed558ccd as int64
    k ^= shr(k, 33)
    k *= -4265267296055464877        # 0xc4ceb9fe1a85ec53 as int64
    k ^= shr(k, 33)
    # unsigned modulo of a value that may have the sign bit set: split off the top bit
    hi = shr(k, 1)
    r = ((hi % mod) * 2 + (k & 1)) % mod
    return r
