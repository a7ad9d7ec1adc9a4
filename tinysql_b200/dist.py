"""Multi-GPU hash join: radix-partition both sides on the join key across the ranks, exchange the partitions, run the
single-GPU join on what arrived.  One process per GPU; torch.distributed is plumbing only (process group, barriers, the NCCL
variant); partitioning, exchange and join are the CUDA kernels of libtinysql_b200.so.

Two exchanges:
  * RegionExchange / RegionJoin (the default of bench.py --gpus N): the scatter kernel stores every row straight into the
    destination rank's receive region over NVLink peer memory (CUDA IPC), chunk by chunk, overlapped with the local join of
    the chunks that have already arrived; device-side epoch flags replace host barriers.
  * exchange() (distributed_join / distributed_agg): partition locally, then ONE grouped NCCL send/recv — the all-to-all at the
    shard boundary (NCCL 2.27/2.28 has no ncclAllToAllv); also what the gloo CPU tests drive.

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


class RegionExchange:
    """The exchange the multi-GPU join runs on: every rank owns ONE device allocation (tq_device_alloc, exported once through
    CUDA IPC and opened by every peer under its own device) that holds, per table t (0 = build side, 1.. = probe chunks):
        slots[t][src] = {u64 rows, u64 epoch}                  16-byte slot per source rank
        region[t][src][col] = cap_t rows x 8 bytes             where source `src` scatters its rows for THIS rank
    A rank pushes table t with tq_partition_push_regions: its scatter kernel stores rows straight into "its" region on every
    peer (NVLink peer stores, no staging, no count exchange first) and then publishes count + epoch in the peer's slot.  The
    receiver enqueues tq_region_wait(slots[t], world, epoch) — a device-side wait — in front of the kernels that read the
    regions and joins them as one segmented batch (tq_join_put_probe_segments): no host round trip and no NCCL call sits
    between the exchange and the join."""

    def __init__(self, lib, L, world, rank, tables, align_rows=4096):
        self.lib, self.L, self.world, self.rank = lib, L, world, rank
        self.ncols = [nc for nc, _ in tables]
        self.cap = [((cap + align_rows - 1) // align_rows) * align_rows for _, cap in tables]
        self.slot_off = [t * world * 16 for t in range(len(tables))]
        off = ((len(tables) * world * 16 + 4095) // 4096) * 4096
        self.reg_off = []
        for nc, cap in zip(self.ncols, self.cap):
            self.reg_off.append(off)
            off += world * nc * cap * 8
        self.total = off
        p = C.c_void_p()
        L.check(lib.tq_device_alloc(self.total, C.byref(p)))
        L.check(lib.tq_memset_device(p, 0, self.total))
        L.check(lib.tq_device_synchronize())
        self.own = p.value
        h = (C.c_ubyte * 64)()
        L.check(lib.tq_ipc_get_handle(p, h))
        gathered = [None] * world
        dist.all_gather_object(gathered, bytes(h))
        self.base, self._opened = [], []
        for d in range(world):
            if d == rank:
                self.base.append(self.own)
                continue
            q = C.c_void_p()
            buf = (C.c_ubyte * 64).from_buffer_copy(gathered[d])
            L.check(lib.tq_ipc_open_handle(buf, C.byref(q)))
            self.base.append(q.value)
            self._opened.append(q.value)
        self.epoch = 0

    def close(self):
        for p in self._opened:
            self.lib.tq_ipc_close_handle(C.c_void_p(p))
        self._opened = []
        dist.barrier()  # nobody frees a buffer a peer still has mapped
        self.lib.tq_device_free(C.c_void_p(self.own))

    def region_ptr(self, dst, t, src, c):
        return self.base[dst] + self.reg_off[t] + ((src * self.ncols[t] + c) * self.cap[t]) * 8

    def slot_ptr(self, dst, t, src):
        return self.base[dst] + self.slot_off[t] + src * 16

    def next_epoch(self):
        self.epoch += 1
        return self.epoch

    def push(self, t, cols, n, slot):
        """scatter this rank's rows of table t into its region on every rank; asynchronous (push stream)"""
        nc, w = self.ncols[t], self.world
        dest = (C.c_void_p * (w * nc))()
        cnts = (C.c_void_p * w)()
        for d in range(w):
            for c in range(nc):
                dest[d * nc + c] = self.region_ptr(d, t, self.rank, c)
            cnts[d] = self.slot_ptr(d, t, self.rank)
        self.L.check(self.lib.tq_partition_push_regions(nc, _tq_cols(self.L, cols, n), 0, n, w, dest, cnts, self.cap[t], slot, self.epoch))

    def wait(self, t):
        """device-side: the compute stream waits until every source has published table t for this epoch"""
        self.L.check(self.lib.tq_region_wait(C.c_void_p(self.slot_ptr(self.rank, t, 0)), self.world, self.epoch))

    def counts(self, t):
        """rows each source wrote into this rank's regions of table t (host read: synchronises the compute stream)"""
        self.wait(t)
        self.L.check(self.lib.tq_compute_synchronize())   # the compute stream only: the pushes of later tables keep running
        raw = np.zeros(2 * self.world, dtype=np.uint64)
        self.L.check(self.lib.tq_memcpy_d2h(raw.ctypes.data, C.c_void_p(self.slot_ptr(self.rank, t, 0)), 16 * self.world))
        cnt = [int(raw[2 * g]) for g in range(self.world)]
        if any(c > self.cap[t] for c in cnt):
            raise RuntimeError(f"region overflow in table {t}: {cnt} rows, capacity {self.cap[t]} (skewed keys)")
        return cnt

    def check_all_counts(self):
        """one host read of every slot of this rank (after the step's joins have consumed the regions): overflow check"""
        nt = len(self.ncols)
        raw = np.zeros(2 * self.world * nt, dtype=np.uint64)
        self.L.check(self.lib.tq_memcpy_d2h(raw.ctypes.data, C.c_void_p(self.slot_ptr(self.rank, 0, 0)), 16 * self.world * nt))
        for t in range(nt):
            cnt = [int(raw[2 * (t * self.world + g)]) for g in range(self.world)]
            if any(c > self.cap[t] for c in cnt):
                raise RuntimeError(f"region overflow in table {t}: {cnt} rows, capacity {self.cap[t]} (skewed keys)")

    def segment_args(self, t):
        """(tq_column array [src][col], count pointer array) of this rank's regions of table t"""
        nc, w = self.ncols[t], self.world
        cols = (self.L.TQColumn * (w * nc))()
        cnts = (C.c_void_p * w)()
        for g in range(w):
            for c in range(nc):
                k = g * nc + c
                cols[k].length, cols[k].data, cols[k].null_bitmap, cols[k].offsets = self.cap[t], self.region_ptr(self.rank, t, g, c), None, None
            cnts[g] = self.slot_ptr(self.rank, t, g)
        return cols, cnts


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
    (nobody may overwrite a region a peer is still joining)."""

    def __init__(self, lib, L, world, rank, n_build_max, n_probe_max, n_chunks, slack=1.25):
        """n_build_max / n_probe_max: the largest per-rank shard (every rank must pass the same numbers: the layout is shared)"""
        self.lib, self.L, self.world, self.rank, self.n_chunks = lib, L, world, rank, n_chunks
        cap = lambda n: int(n / world * slack) + (1 << 14)   # keys are hash-spread: +25 % covers the imbalance between (source, destination) pairs
        chunk_max = (n_probe_max + n_chunks - 1) // n_chunks
        tables = [(2, cap(n_build_max))] + [(2, cap(chunk_max)) for c in range(n_chunks)]
        self.rx = RegionExchange(lib, L, world, rank, tables)

    def close(self):
        self.rx.close()

    def step(self, bk, bv, pk, pv, keep_result=False):
        """bk / bv / pk / pv: this rank's row shards as (device pointer, rows)-like objects.  Returns (rows, stats, result)."""
        lib, L, rx, w = self.lib, self.L, self.rx, self.world
        t_start = time.perf_counter()
        trace = []
        mark = lambda name: trace.append((name, (time.perf_counter() - t_start) * 1e3))   # host-side timeline: where the host blocks
        n_probe = int(pk.numel())
        bounds = [n_probe * i // self.n_chunks for i in range(self.n_chunks + 1)]
        rx.next_epoch()
        rx.push(0, [bk, bv], int(bk.numel()), 0)
        for c in range(self.n_chunks):
            lo, hi = bounds[c], bounds[c + 1]
            rx.push(1 + c, [RawCol(pk.data_ptr() + lo * 8, hi - lo), RawCol(pv.data_ptr() + lo * 8, hi - lo)], hi - lo, 1 + c)
        mark("pushes enqueued")
        # ---- build side: the only place the host needs row counts
        cnt_b = rx.counts(0)
        mark("build rows arrived (host read)")
        t = (C.c_int32 * 2)(1, 1)
        k = (C.c_int32 * 1)(0)
        d = L.TQJoinDesc(0, 1, 2, t, 2, t, 1, k, k, 0, 0)
        h = C.c_void_p()
        L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
        total, result, st = 0, None, (C.c_int64 * 8)()
        try:
            for g in range(w):
                if cnt_b[g]:
                    cols = [RawCol(rx.region_ptr(self.rank, 0, g, c), cnt_b[g]) for c in range(2)]
                    L.check(lib.tq_join_put_build(h, _tq_cols(L, cols, cnt_b[g]), L.TQ_MEM_DEVICE))
            L.check(lib.tq_join_finalize_build(h))
            mark("build done")
            out = (L.TQColumn * 4)()
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
                        chunks.append([device_to_host(1, out[c].data, None, n.value).values for c in range(4)])
                    if not final:
                        return
            for c in range(self.n_chunks):
                rx.wait(1 + c)                                   # device-side: chunk c has landed from every source
                cols, cnts = rx.segment_args(1 + c)
                st_ = lib.tq_join_put_probe_segments(h, w, cols, cnts, rx.cap[1 + c])
                L.check(st_)
                mark(f"chunk {c} enqueued")
                if c >= 1:
                    drain(False)                                 # hand back the batch before last (keeps two result sets alive, not n_chunks)
                    mark(f"chunk {c - 1} drained")
            L.check(lib.tq_join_probe_eof(h))
            drain(True)
            mark("all drained")
            lib.tq_join_stats(h, st)
            if keep_result:
                result = [np.concatenate([ch[c] for ch in chunks]) if chunks else np.zeros(0, np.int64) for c in range(4)]
        finally:
            lib.tq_join_destroy(h)
        rx.check_all_counts()                                    # a region overflow would have dropped rows: fail loudly
        mark("overflow checks")
        dist.barrier()
        mark("barrier")
        self.last_trace = trace
        return total, list(st), result


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
