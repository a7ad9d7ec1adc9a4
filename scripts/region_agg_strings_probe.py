"""Cost of a string GROUP BY over the region exchange next to the same GROUP BY on an INT64 key, on the per-rank C4 shape:
--rows rows per rank (2e7 by default), keys uniform over --keys distinct values (1e6), SUM(x), COUNT(*) and FIRSTROW(k).  The
VARCHAR key is 'k' followed by 10 digits (11 bytes); the INT64 key is the number behind it.  W ranks are emulated on ONE GPU
in this process (every rank's regions in this GPU's memory, dist.RegionAgg.table_of's layout), both variants through
dist.RegionAgg's calls (tq_agg_push_partial_var / tq_agg_merge_regions_var).  Per source: the partial aggregation
(tq_agg_put + tq_agg_eof) and the push (export, destination, scatter, publish); per destination: the merge (tq_region_wait +
merge) and the final (tq_agg_eof + tq_agg_next_device).  Each phase is host time around calls that end in a device
synchronise; bytes pushed = rows published x 8-byte words (+ 8 per string column's offset) + the cells.  NVLink time is not
measured: the regions are local.

Prints one JSON line with the card name and power limit read in the same run.

    python scripts/region_agg_strings_probe.py [--ranks 2] [--rows 20000000] [--keys 1000000] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COUNT, SUM, FIRSTROW = 0, 1, 5
FUNCS = [(SUM, 1), (COUNT, -1), (FIRSTROW, 0)]
KEY_BYTES = 11


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def shard(torch, dev, seed, n, n_keys, strings):
    """(k, x) on the device: k an INT64 tensor, or a VarCol over 'k%010d' cells and the tensors that hold them"""
    from tinysql_b200.dist import VarCol
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    k = torch.randint(0, n_keys, (n,), device=dev, generator=g, dtype=torch.int64)
    x = torch.randint(-1000, 1000, (n,), device=dev, generator=g, dtype=torch.int64)
    if not strings:
        return [k, x], []
    p10 = torch.tensor([10 ** (9 - j) for j in range(10)], dtype=torch.int64, device=dev)
    cells = torch.empty((n, KEY_BYTES), dtype=torch.uint8, device=dev)
    cells[:, 0] = ord("k")
    cells[:, 1:] = ((k[:, None] // p10) % 10 + ord("0")).to(torch.uint8)
    off = torch.arange(0, (n + 1) * KEY_BYTES, KEY_BYTES, dtype=torch.int64, device=dev)
    return [VarCol(cells.data_ptr(), off.data_ptr(), n), x], [cells, off, k]


def timed(lib, L, fn):
    t0 = time.perf_counter()
    fn()
    L.check(lib.tq_device_synchronize())
    return (time.perf_counter() - t0) * 1e3


def variant(torch, lib, L, dev, args, strings):
    """W emulated ranks: per-phase ms (mean over sources / destinations, best rep), groups and bytes pushed per rank"""
    import broadcast_ref as B
    from tinysql_b200.dist import RegionAgg
    W = args.ranks
    types = [L.TQ_TYPE_BYTES if strings else L.TQ_TYPE_INT64, L.TQ_TYPE_INT64]
    caps = [args.keys * KEY_BYTES, None] if strings else None
    from tinysql_b200.dist import _tq_device, partial_var_cols
    width = len(FUNCS) + 1
    table, _ = RegionAgg.table_of(W, width, partial_var_cols(types, [0], FUNCS), True, args.keys, caps)
    ex = B.EmuExchange(lib, W, table)
    aggs = [RegionAgg(lib, L, W, r, types, [0], FUNCS, args.keys, est_groups=args.keys, slot=r, byte_caps=caps, exchange=B.RankView(ex, r))
            for r in range(W)]
    data = [shard(torch, dev, 1000 * (1 + strings) + s, args.rows, args.keys, strings) for s in range(W)]
    torch.cuda.synchronize()
    best, groups, pushed = None, 0, 0
    for rep in range(args.reps + 1):
        ex.next_epoch()
        ph = {"partial_agg": [], "push": [], "merge": [], "final": []}
        for s, a in enumerate(aggs):
            cols = data[s][0]
            # RegionAgg.push's three calls, timed apart: put + eof, then the push
            arr, n = _tq_device(L, cols)
            h, _ = a._create()
            ph["partial_agg"].append(timed(lib, L, lambda: (L.check(lib.tq_agg_put(h, arr, L.TQ_MEM_DEVICE)), L.check(lib.tq_agg_eof(h)))))
            a._hp = h
            dest, cnts = ex.push_tables(0, s)
            bc = (C.c_int64 * max(len(a.byte_cap), 1))(*a.byte_cap)
            ph["push"].append(timed(lib, L, lambda: (L.check(lib.tq_agg_push_partial_var(h, W, dest, cnts, ex.cap[0], bc, s, ex.epoch)),
                                                      L.check(lib.tq_partition_push_sync(s)))))
        groups, pushed = 0, 0
        for q, a in enumerate(aggs):
            hf, _ = a._create()
            regs, slots = a.merge_table(q), C.c_void_p(ex.slot_ptr(q, 0, 0))
            ph["merge"].append(timed(lib, L, lambda: (a.rx.wait(0), L.check(lib.tq_agg_merge_regions_var(hf, W, slots, ex.cap[0], regs)))))
            out = (L.TQColumn * 3)()
            n, eof = C.c_int64(0), C.c_int32(0)
            ph["final"].append(timed(lib, L, lambda: (L.check(lib.tq_agg_eof(hf)), L.check(lib.tq_agg_next_device(hf, out, C.byref(n), C.byref(eof))))))
            groups += n.value
            rows = [int(r) for r in ex.read_slots(q)[0][:, 0]]
            pushed += sum(rows) * (a.width + 1 + len(a.var_cols)) * 8
            for g in range(W):
                for v, (c, _) in enumerate(a.var_cols):
                    last = np.zeros(1, np.int64)
                    if rows[g]:
                        L.check(lib.tq_memcpy_d2h(last.ctypes.data, C.c_void_p(ex.region_ptr(q, 0, g, c) + rows[g] * 8), 8))
                    pushed += int(last[0])
            lib.tq_agg_destroy(hf)
        for a in aggs:
            lib.tq_agg_destroy(a._hp)
            a._hp = None
        if rep == 0:
            continue                                                     # warm-up: module load, table growth
        mean = {k: float(np.mean(v)) for k, v in ph.items()}
        if best is None or sum(mean.values()) < sum(best.values()):
            best = mean
    ex.free()
    del data
    torch.cuda.empty_cache()
    return {"ms_per_rank": {k: round(v, 3) for k, v in best.items()}, "groups": groups, "bytes_pushed_per_rank": pushed // W,
            "wire_areas": table[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=2, help="emulated ranks on one GPU")
    ap.add_argument("--rows", type=int, default=20_000_000)
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    from tinysql_b200 import _lib as L
    lib = L.load()
    L.check(lib.tq_init(0))
    dev = torch.device("cuda", 0)
    res = {"card": card(), "rows_per_rank": args.rows, "keys": args.keys, "ranks_emulated": args.ranks,
           "note": "mean over the sources (partial_agg, push) or destinations (merge, final); best of the reps; NVLink not measured"}
    for name, strings in (("int64_key", False), ("varchar_key", True)):
        res[name] = variant(torch, lib, L, dev, args, strings)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
