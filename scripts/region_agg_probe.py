"""Cost of the GROUP BY over the region exchange on the per-rank C4 shape: 1e8 rows per rank, keys uniform in [0, 1e6),
SUM(x) and COUNT(*) (plus FIRSTROW(k), which names each result row's group), in two variants: NOT NULL, and nullable with 5 %
NULL x and 1 % NULL keys.

  emulated : W ranks on ONE GPU in this process (every rank's regions in this GPU's memory: tests/exchange_ref.py's Regions,
             with dist.RegionLayout's argument tables).  Per source: the partial
             aggregation (tq_agg_put + tq_agg_eof) and the push (tq_agg_push_partial: export, destination, scatter, publish);
             per destination: the merge (tq_region_wait + tq_agg_merge_regions) and the final (tq_agg_eof + tq_agg_next_device).
             Each phase is host time around calls that end in a device synchronise; bytes pushed from the published slots.
  group    : dist.RegionAgg over the process group (torchrun: one rank per GPU; plain python: a group of one), and, on the NOT NULL
             variant, the NCCL path (distributed_agg + gpu_agg_fns) on the same shard: step times and equal results.

Prints one JSON line per rank 0 with the card name and power limit.

    python scripts/region_agg_probe.py [--ranks 2] [--rows 100000000] [--keys 1000000] [--reps 3]
    torchrun --nproc-per-node=N scripts/region_agg_probe.py ...
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def shard(torch, dev, seed, n, n_keys, nullable):
    """(k, x) on the device and their NULL bitmaps (None for NOT NULL)"""
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    k = torch.randint(0, n_keys, (n,), device=dev, generator=g, dtype=torch.int64)
    x = torch.randint(-1000, 1000, (n,), device=dev, generator=g, dtype=torch.int64)
    if not nullable:
        return [k, x], None
    w = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.int64, device=dev)

    def bitmap(p_null):
        nn = (torch.rand(((n + 63) // 64) * 64, device=dev, generator=g) >= p_null).to(torch.int64)
        return torch.cat([(nn.view(-1, 8) * w).sum(1).to(torch.uint8), torch.zeros(8, dtype=torch.uint8, device=dev)])
    return [k, x], [bitmap(0.01), bitmap(0.05)]


def timed(lib, L, fn):
    t0 = time.perf_counter()
    fn()
    L.check(lib.tq_device_synchronize())
    return (time.perf_counter() - t0) * 1e3


def emulated(torch, lib, L, D, dev, args, nullable):
    """W ranks on this GPU: per-phase ms (mean over sources / destinations, best rep) and bytes pushed"""
    import exchange_ref as X
    W = args.ranks
    t = L.TQ_TYPE_INT64 if nullable else L.TQ_TYPE_INT64 | L.TQ_TYPE_NOT_NULL
    it = (C.c_int32 * 2)(t, t)
    gb = (C.c_int32 * 1)(0)
    fa = (L.TQAggFunc * 3)(*[L.TQAggFunc(f, a) for f, a in FUNCS])
    d = L.TQAggDesc(2, it, 1, gb, 3, fa, args.keys)

    def create():
        h = C.c_void_p()
        L.check(lib.tq_agg_create(C.byref(d), C.byref(h)))
        return h
    h = create()
    wd = C.c_int32(0)
    L.check(lib.tq_agg_partial_width(h, C.byref(wd)))
    lib.tq_agg_destroy(h)
    nw = wd.value + 1
    cap = int(args.keys / W * 1.25) + (1 << 14)
    reg = X.Regions(lib, W, nw, cap, guard=0)
    data = [shard(torch, dev, 1000 * (1 + nullable) + s, args.rows, args.keys, nullable) for s in range(W)]
    torch.cuda.synchronize()
    best, groups, pushed = None, 0, 0
    for rep in range(args.reps + 1):
        epoch = rep + 1
        ph = {"partial_agg": [], "push": [], "merge": [], "final": []}
        hs = []
        for s in range(W):
            cols, bms = data[s]
            arr = D._tq_cols(L, cols, args.rows)
            for c, b in enumerate(bms or []):
                arr[c].null_bitmap = b.data_ptr()
            h = create()
            hs.append(h)
            ph["partial_agg"].append(timed(lib, L, lambda: (L.check(lib.tq_agg_put(h, arr, L.TQ_MEM_DEVICE)), L.check(lib.tq_agg_eof(h)))))
            dest, cnts = reg.push_tables(0, s)
            ph["push"].append(timed(lib, L, lambda: (L.check(lib.tq_agg_push_partial(h, W, dest, cnts, cap, s, epoch)),
                                                      L.check(lib.tq_partition_push_sync(s)))))
        groups, pushed = 0, 0
        for q in range(W):
            hf = create()
            regs, slots = reg.region_table(q, 0), C.c_void_p(reg.slot_ptr(q, 0, 0))
            ph["merge"].append(timed(lib, L, lambda: (L.check(reg.wait(q, epoch)), L.check(lib.tq_agg_merge_regions(hf, W, slots, cap, regs)))))
            out = (L.TQColumn * 3)()
            n, eof = C.c_int64(0), C.c_int32(0)
            ph["final"].append(timed(lib, L, lambda: (L.check(lib.tq_agg_eof(hf)), L.check(lib.tq_agg_next_device(hf, out, C.byref(n), C.byref(eof))))))
            groups += n.value
            pushed += sum(rows for rows, _ in reg.slots(q)) * nw * 8
            lib.tq_agg_destroy(hf)
        for h in hs:
            lib.tq_agg_destroy(h)
        if rep == 0:
            continue                                                     # warm-up: module load, table growth
        mean = {k: float(np.mean(v)) for k, v in ph.items()}
        if best is None or sum(mean.values()) < sum(best.values()):
            best = mean
    reg.free()
    del data
    torch.cuda.empty_cache()
    return {"ranks_emulated": W, "ms_per_rank": {k: round(v, 3) for k, v in best.items()}, "groups": groups,
            "bytes_pushed_per_rank": pushed // W, "wire_words_per_row": nw,
            "input_bytes_per_rank": args.rows * 16, "note": "mean over the sources (partial_agg, push) or destinations (merge, final); best of the reps"}


def group_runs(torch, lib, L, D, dist, dev, args, rank, world):
    """RegionAgg over the process group on both variants, the NCCL path on the NOT NULL one; results compared"""
    import region_agg_ref as RA
    out = {}
    for nullable in (False, True):
        cols, bms = shard(torch, dev, 7000 * (1 + nullable) + rank, args.rows, args.keys, nullable)
        types = [L.TQ_TYPE_INT64] * 2 if nullable else [L.TQ_TYPE_INT64 | L.TQ_TYPE_NOT_NULL] * 2
        ra = D.RegionAgg(lib, L, world, rank, types, [0], FUNCS, args.keys, est_groups=args.keys, slot=0)
        times = []
        res = None
        for rep in range(args.reps + 1):
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            _, res = ra.step(cols, [b.data_ptr() for b in bms] if bms else None, keep_result=(rep == args.reps))
            times.append((time.perf_counter() - t0) * 1e3)
        ra.close()
        key = "nullable" if nullable else "not_null"
        out[key] = {"region_step_ms": round(float(np.min(times[1:])), 3), "groups_rank": int(res[0].length)}
        if not nullable:
            partial_fn, final_fn = D.gpu_agg_fns(lib, L, [L.TQ_TYPE_INT64] * 2, 0, FUNCS, est_groups=args.keys)
            nt, nres = [], None
            for rep in range(args.reps + 1):
                torch.cuda.synchronize()
                dist.barrier()
                t0 = time.perf_counter()
                nres = D.distributed_agg(cols, world, rank, partial_fn, D.gpu_partition_fn(lib, L), final_fn)
                torch.cuda.synchronize()
                nt.append((time.perf_counter() - t0) * 1e3)
            out[key]["nccl_step_ms"] = round(float(np.min(nt[1:])), 3)
            out[key]["equal_to_nccl"] = bool(np.array_equal(RA.canon(res), RA.canon(nres)))
        del cols, bms
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=2, help="emulated ranks on one GPU (plain python runs only)")
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    import torch.distributed as dist

    from tinysql_b200 import _lib as L
    from tinysql_b200 import dist as D
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    if "RANK" not in os.environ:
        os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": "29523", "RANK": "0", "WORLD_SIZE": "1"})
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    lib = L.load()
    L.check(lib.tq_init(local))
    dev = torch.device("cuda", local)
    res = {"card": card(), "rows_per_rank": args.rows, "keys": args.keys, "world": world}
    if world == 1:
        res["emulated"] = {v: emulated(torch, lib, L, D, dev, args, v == "nullable") for v in ("not_null", "nullable")}
    res["group"] = group_runs(torch, lib, L, D, dist, dev, args, rank, world)
    if rank == 0:
        print(json.dumps(res), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
