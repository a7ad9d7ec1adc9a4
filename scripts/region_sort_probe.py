"""Cost of the multi-GPU ORDER BY (dist.RegionSort) with W ranks emulated on ONE GPU, next to the single-GPU tq_sort of the
same rows.  Two shapes: --rows rows per rank (1e8 by default) of an INT64 key with an INT64 payload, and --str-rows rows per
rank (2e7) of an 11-byte VARCHAR key ('k' + 10 digits) with an INT64 payload; keys uniform.  Every rank's regions sit in
this GPU's memory (RegionSort.table_of's layout), so NVLink time is not measured.

Per phase, host time around calls that end in a device synchronise, summed over the emulated ranks: sample (every rank's
tq_partition_push_sample), push (every rank's splitters — tq_region_wait, the sort of the W samples — and
tq_partition_push_ranges), wait + put (tq_region_wait + tq_sort_put_regions), sort (tq_sort_eof), drain
(tq_sort_next_device).  Bytes pushed = rows x (8 per column + 8 for the mask word) + the cells.  Beside them: the single-GPU
tq_sort of all ranks' rows (device puts, eof, next_device).  Prints one JSON line per shape with the card name and power
limit read in the same run.

    python scripts/region_sort_probe.py [--ranks 2] [--rows 100000000] [--str-rows 20000000] [--reps 2]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KEY_BYTES = 11


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def shard(torch, dev, seed, n, strings):
    """(key, payload) on the device: an INT64 key, or a VarCol over 'k%010d' cells"""
    from tinysql_b200.dist import VarCol
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    k = torch.randint(0, 1 << 40, (n,), device=dev, generator=g, dtype=torch.int64)
    x = torch.arange(n, device=dev, dtype=torch.int64)
    if not strings:
        return [k, x], [k, x]
    k = k % 10_000_000_000
    p10 = torch.tensor([10 ** (9 - j) for j in range(10)], dtype=torch.int64, device=dev)
    cells = torch.empty((n, KEY_BYTES), dtype=torch.uint8, device=dev)
    cells[:, 0] = ord("k")
    cells[:, 1:] = ((k[:, None] // p10) % 10 + ord("0")).to(torch.uint8)
    off = torch.arange(0, (n + 1) * KEY_BYTES, KEY_BYTES, dtype=torch.int64, device=dev)
    del k
    return [VarCol(cells.data_ptr(), off.data_ptr(), n), x], [cells, off, x]


def timed(lib, L, fn):
    t0 = time.perf_counter()
    fn()
    L.check(lib.tq_device_synchronize())
    return (time.perf_counter() - t0) * 1e3


def one_gpu(lib, L, types, data):
    """the single-GPU tq_sort of every rank's rows: (ms, rows)"""
    from tinysql_b200.dist import _tq_device
    tt = (C.c_int32 * 2)(*types)
    bc, bd = (C.c_int32 * 1)(0), (C.c_int32 * 1)(0)
    d = L.TQSortDesc(2, tt, 1, bc, bd, 0, -1)
    h = C.c_void_p()
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    out, rows, eof = (L.TQColumn * 2)(), C.c_int64(0), C.c_int32(0)
    try:
        def run():
            for cols, _ in data:
                L.check(lib.tq_sort_put(h, _tq_device(L, cols)[0], L.TQ_MEM_DEVICE))
            L.check(lib.tq_sort_eof(h))
            L.check(lib.tq_sort_next_device(h, out, C.byref(rows), C.byref(eof)))
        return timed(lib, L, run), rows.value
    finally:
        lib.tq_sort_destroy(h)


def variant(torch, lib, L, dev, W, n, reps, strings):
    import region_sort_ref as RS
    types = [L.TQ_TYPE_BYTES if strings else L.TQ_TYPE_INT64, L.TQ_TYPE_INT64]
    caps = [n * KEY_BYTES, None] if strings else None
    em = RS.Emulated(lib, W, types, [0], [False], n, caps, False)
    data = [shard(torch, dev, 7000 * (1 + strings) + s, n, strings) for s in range(W)]
    torch.cuda.synchronize()
    best, rows_per_rank = None, []
    try:
        for rep in range(reps + 1):
            em.ex.next_epoch()
            ph = {}
            ph["sample"] = timed(lib, L, lambda: [em.sorts[r].push_sample(data[r][0]) for r in range(W)])
            ph["push"] = timed(lib, L, lambda: [em.sorts[r].push_rows(data[r][0]) for r in range(W)])
            ph["wait + put"] = ph["sort"] = ph["drain"] = 0.0
            rows_per_rank = []
            for r in range(W):
                s = em.sorts[r]
                rx = s.rx
                h = s._sort(2, types, [0], [0], 0, -1)
                regs = (L.TQColumn * (W * 3))()
                for g in range(W):
                    for c in range(3):
                        regs[g * 3 + c].length, regs[g * 3 + c].data = rx.cap[1], rx.region_ptr(r, 1, g, c)
                    if strings:
                        regs[g * 3].offsets, regs[g * 3].data = regs[g * 3].data, rx.region_ptr(r, 1, g, 3)

                def put():
                    rx.wait(1)
                    L.check(lib.tq_sort_put_regions(h, W, C.c_void_p(rx.slot_ptr(r, 1, 0)), rx.cap[1], regs))
                ph["wait + put"] += timed(lib, L, put)
                ph["sort"] += timed(lib, L, lambda: L.check(lib.tq_sort_eof(h)))
                got = []
                ph["drain"] += timed(lib, L, lambda: got.append(s._lend(h, 2)[1]))
                rows_per_rank.append(got[0])
            for s in em.sorts:
                s.release()
            ph["total"] = sum(ph.values())
            if rep and (best is None or ph["total"] < best["total"]):
                best = ph
        single = min(one_gpu(lib, L, types, data)[0] for _ in range(reps))
    finally:
        for s in em.sorts:
            s.release()
        em.free()
    pushed = sum(rows_per_rank) * (3 * 8) + (W * n * KEY_BYTES if strings else 0)
    return {"shape": f"{'VARCHAR(11)' if strings else 'INT64'} key + INT64 payload", "ranks": W, "rows_per_rank": n,
            "ms": {k: round(v, 2) for k, v in best.items()}, "rows_received": rows_per_rank, "bytes_pushed": pushed,
            "one_gpu_tq_sort_ms": round(single, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=2)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--str-rows", type=int, default=20_000_000)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import torch
    from tinysql_b200 import _lib as L
    lib = L.load()
    L.check(lib.tq_init(0))
    dev = torch.device("cuda", 0)
    gpu = card()
    for strings, n in ((False, args.rows), (True, args.str_rows)):
        res = variant(torch, lib, L, dev, args.ranks, n, args.reps, strings)
        res["card"] = gpu
        print(json.dumps(res), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
