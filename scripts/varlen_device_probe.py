"""Var-len columns from host memory vs from HBM, end to end through the C-ABI.

Join (BASELINE C1, the reference's executor/benchmark_test.go:391-457 shape at full size): 2 x 1e5 rows of (BIGINT k = row,
5 KiB VARSTRING), inner join on keys {0, 1}, then on {0}.  Three arms, wall time of the handle from tq_join_create to the last
result batch:
  (a) host chunks of <= 1024 rows (the chunk protocol), results read with tq_join_next;
  (b) one large host column per side, results read with tq_join_next;
  (c) wire bytes (chunk.Codec) -> tq_chunk_decode_device -> TQ_MEM_DEVICE puts -> tq_join_next_device (results stay in HBM).
GROUP BY a VARCHAR column (1e7 rows, 1e5 distinct strings; COUNT(*), FIRSTROW): host chunks vs wire chunks decoded on the
device, both 1024 rows per chunk, results lent by tq_agg_next_device.

Every output row is checked (join: both keys equal and each string is the function of its key; aggregation: every group's
count and value).  Bytes over PCIe are computed from the shapes.  Prints the card's name and power limit read in the same run,
then one JSON line.  Needs a GPU: there is no CPU fallback."""
import ctypes as C
import json
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import BYTES, INT64, Column, DeviceChunk, VarColumn, encode_chunk, tq_array
from tinysql_b200.executor import AGG_COUNT, AGG_FIRSTROW

REPS, CELL, ROWS = 5, 5120, 100_000
lib = L.load()
L.check(lib.tq_init(0))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def var_column(offsets, data):
    c = object.__new__(VarColumn)
    c.tp, c.length, c.offsets, c.data, c.bitmap = BYTES, len(offsets) - 1, np.ascontiguousarray(offsets, np.int64), np.ascontiguousarray(data, np.uint8), None
    return c


def i32(v):
    return (C.c_int32 * len(v))(*v)


def d2h(ptr, nbytes, dtype):
    out = np.empty(nbytes // np.dtype(dtype).itemsize, dtype=dtype)
    if nbytes:
        L.check(lib.tq_memcpy_d2h(out.ctypes.data, ptr, nbytes))
    return out


def median_time(fn):
    fn()                                          # warm-up: allocations, module load
    ts = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts), ts


# ---------------------------------------------------------------------------------------------------- join (C1)
k = np.arange(ROWS, dtype=np.int64)
cells = np.repeat(k, CELL // 8).view(np.uint8)    # cell of row r = 640 copies of r: the string is a function of the key
side = [Column(INT64, k), var_column(np.arange(ROWS + 1, dtype=np.int64) * CELL, cells)]
types = [INT64, BYTES]


def side_view(lo, hi):
    """tq_columns of rows [lo, hi) of one side, pointing into the side's buffers (offsets[0] = lo * CELL)"""
    arr = (L.TQColumn * 2)()
    arr[0] = L.TQColumn(hi - lo, None, None, k.ctypes.data + lo * 8)
    arr[1] = L.TQColumn(hi - lo, None, side[1].offsets.ctypes.data + lo * 8, side[1].data.ctypes.data)
    return arr


def side_slice(lo, hi):
    return [Column(INT64, k[lo:hi]), var_column(side[1].offsets[lo: hi + 1] - side[1].offsets[lo], cells[lo * CELL: hi * CELL])]


def check_join_rows(pk, ps_off, ps, bk, bs_off, bs):
    """output (P.k, P.s, B.k, B.s): keys equal, every string = its key repeated, every key exactly once"""
    m = len(pk)
    assert m == ROWS and np.array_equal(pk, bk) and np.array_equal(np.sort(pk), k)
    for off, data in ((ps_off, ps), (bs_off, bs)):
        assert np.array_equal(off - off[0], np.arange(m + 1, dtype=np.int64) * CELL)
        assert np.array_equal(data.view(np.int64).reshape(m, CELL // 8), np.repeat(pk, CELL // 8).reshape(m, CELL // 8))


def join_host(keys, piece, verify=False):
    d = L.TQJoinDesc(0, 0, 2, i32(types), 2, i32(types), len(keys), i32(keys), i32(keys), 0, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    for lo in range(0, ROWS, piece):
        L.check(lib.tq_join_put_build(h, side_view(lo, min(ROWS, lo + piece)), L.TQ_MEM_HOST))
    L.check(lib.tq_join_finalize_build(h))
    for lo in range(0, ROWS, piece):
        L.check(lib.tq_join_put_probe(h, side_view(lo, min(ROWS, lo + piece)), None, L.TQ_MEM_HOST))
    L.check(lib.tq_join_probe_eof(h))
    req = min(piece, ROWS)
    got = [[], [], [], []]
    n, eof = C.c_int64(0), C.c_int32(0)
    need = (C.c_int64 * 4)()
    while True:
        L.check(lib.tq_join_next_bytes(h, req, need))
        out = [Column.empty(INT64, req), VarColumn.empty(BYTES, req, need[1]), Column.empty(INT64, req), VarColumn.empty(BYTES, req, need[3])]
        L.check(lib.tq_join_next(h, req, tq_array(out, req), C.byref(n), C.byref(eof)))
        if n.value == 0 and eof.value:
            break
        if verify and n.value:
            m = n.value
            got[0].append(out[0].values[:m].copy()); got[2].append(out[2].values[:m].copy())
            got[1].append(out[1].data[: out[1].offsets[m]].copy()); got[3].append(out[3].data[: out[3].offsets[m]].copy())
    L.check(lib.tq_join_destroy(h))
    if verify:
        pk, bk = np.concatenate(got[0]), np.concatenate(got[2])
        offs = np.arange(len(pk) + 1, dtype=np.int64) * CELL
        check_join_rows(pk, offs, np.concatenate(got[1]), bk, offs, np.concatenate(got[3]))


wire_side = [encode_chunk(types, side_slice(lo, min(ROWS, lo + 1024))) for lo in range(0, ROWS, 1024)]


def join_device(keys, verify=False):
    d = L.TQJoinDesc(0, 0, 2, i32(types), 2, i32(types), len(keys), i32(keys), i32(keys), 0, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    build = [DeviceChunk().decode(w, types) for w in wire_side]   # 8-byte build columns are borrowed until finalize_build
    for dc in build:
        L.check(lib.tq_join_put_build(h, dc.tq_cols, L.TQ_MEM_DEVICE))
    L.check(lib.tq_join_finalize_build(h))
    for dc in build:
        dc.free()
    out = (L.TQColumn * 4)()
    n, eof = C.c_int64(0), C.c_int32(0)
    got = []

    def drain():
        while True:
            L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
            if n.value == 0:
                return
            if verify:
                m = n.value
                po, bo = d2h(out[1].offsets, (m + 1) * 8, np.int64), d2h(out[3].offsets, (m + 1) * 8, np.int64)
                got.append((d2h(out[0].data, m * 8, np.int64), po, d2h(out[1].data + int(po[0]), int(po[m] - po[0]), np.uint8),
                            d2h(out[2].data, m * 8, np.int64), bo, d2h(out[3].data + int(bo[0]), int(bo[m] - bo[0]), np.uint8)))

    dp = DeviceChunk()
    for w in wire_side:
        dp.decode(w, types)
        L.check(lib.tq_join_put_probe(h, dp.tq_cols, None, L.TQ_MEM_DEVICE))
        drain()                                   # the batch that borrowed dp's columns is finished before dp is reused
    L.check(lib.tq_join_probe_eof(h))
    drain()
    dp.free()
    L.check(lib.tq_join_destroy(h))
    if verify:
        pk = np.concatenate([g[0] for g in got])
        offs = np.arange(len(pk) + 1, dtype=np.int64) * CELL
        for g in got:
            m = len(g[0])
            assert np.array_equal(g[1] - g[1][0], offs[: m + 1]) and np.array_equal(g[4] - g[4][0], offs[: m + 1])
        check_join_rows(pk, offs, np.concatenate([g[2] for g in got]), np.concatenate([g[3] for g in got]), offs, np.concatenate([g[5] for g in got]))


side_bytes = ROWS * 8 + ROWS * CELL + (ROWS + 1) * 8                   # k + cells + offsets
out_bytes = ROWS * (8 + 8) + 2 * ROWS * CELL + 2 * (ROWS + 1) * 8 + 4 * ((ROWS + 7) // 8)
wire_bytes = sum(len(w) for w in wire_side)
name, power = card()
print(f"card: {name}, power limit {power}", flush=True)
results = {"card": name, "power_limit": power, "join": [], "group_by": []}
for keys in ([0, 1], [0]):
    for arm, fn, h2d, d2h_b in (("a: host chunks <= 1024 rows", lambda v=False: join_host(keys, 1024, v), 2 * side_bytes, out_bytes),
                                ("b: one host column per side", lambda v=False: join_host(keys, ROWS, v), 2 * side_bytes, out_bytes),
                                ("c: wire bytes -> device decode -> device puts -> lent results", lambda v=False: join_device(keys, v), 2 * wire_bytes, 0)):
        fn(True)                                  # every output row checked
        med, ts = median_time(fn)
        results["join"].append({"keys": keys, "arm": arm, "median_s": med, "runs_s": ts, "h2d_bytes": h2d, "d2h_bytes": d2h_b, "rows_checked": ROWS})
        print(json.dumps(results["join"][-1]), flush=True)

# ---------------------------------------------------------------------------------------------------- GROUP BY VARCHAR
N, G = 10_000_000, 100_000
rng = np.random.default_rng(3)
gid = rng.integers(0, G, N)
gcells = np.stack([gid, gid * 2654435761 + 7], axis=1).reshape(-1).view(np.uint8)   # 16-byte cell of group g: (g, h(g))
gcol = var_column(np.arange(N + 1, dtype=np.int64) * 16, gcells)
want_count = np.bincount(gid, minlength=G)
at = [BYTES]
funcs = [(AGG_COUNT, -1), (AGG_FIRSTROW, 0)]


def agg_run(device, verify=False):
    fa = (L.TQAggFunc * 2)(*[L.TQAggFunc(f, a) for f, a in funcs])
    d = L.TQAggDesc(1, i32(at), 1, i32([0]), 2, fa, G)
    h = C.c_void_p()
    L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
    if device:
        dc = DeviceChunk()
        for w in wire_agg:
            dc.decode(w, at)
            L.check(lib.tq_agg_put(h, dc.tq_cols, L.TQ_MEM_DEVICE))
        dc.free()
    else:
        for lo in range(0, N, 1024):
            hi = min(N, lo + 1024)
            t = L.TQColumn(hi - lo, None, gcol.offsets.ctypes.data + lo * 8, gcol.data.ctypes.data)
            L.check(lib.tq_agg_put(h, (L.TQColumn * 1)(t), L.TQ_MEM_HOST))
    L.check(lib.tq_agg_eof(h))
    out = (L.TQColumn * 2)()
    n, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_agg_next_device(h, out, C.byref(n), C.byref(eof)))
    if verify:
        m = n.value
        assert m == np.count_nonzero(want_count)
        cnt = d2h(out[0].data, m * 8, np.int64)
        off = d2h(out[1].offsets, (m + 1) * 8, np.int64)
        assert np.array_equal(off - off[0], np.arange(m + 1, dtype=np.int64) * 16)
        v = d2h(out[1].data + int(off[0]), m * 16, np.uint8).view(np.int64).reshape(m, 2)
        assert np.array_equal(v[:, 1], v[:, 0] * 2654435761 + 7)
        assert np.array_equal(cnt, want_count[v[:, 0]]) and len(np.unique(v[:, 0])) == m
    L.check(lib.tq_agg_destroy(h))


wire_agg = [encode_chunk(at, [var_column(gcol.offsets[lo: min(N, lo + 1024) + 1] - gcol.offsets[lo], gcells[lo * 16: min(N, lo + 1024) * 16])])
            for lo in range(0, N, 1024)]
for arm, dev, h2d in (("host chunks of 1024 rows", False, N * 16 + (N + 1) * 8), ("wire chunks of 1024 rows decoded on the device", True, sum(len(w) for w in wire_agg))):
    agg_run(dev, True)
    med, ts = median_time(lambda: agg_run(dev))
    results["group_by"].append({"arm": arm, "rows": N, "groups": G, "median_s": med, "runs_s": ts, "h2d_bytes": h2d, "groups_checked": G})
    print(json.dumps(results["group_by"][-1]), flush=True)
print(json.dumps({"varlen_device_probe": results}))
