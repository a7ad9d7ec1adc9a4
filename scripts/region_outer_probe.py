"""Cost of the outer-join / nullable path of the region exchange on ONE GPU with W emulated ranks (all receive buffers in
this GPU's memory), on the per-rank C5 shape (12.5M build / 125M probe rows per rank by default, uniform keys, every probe row
matches once).  W sources push into one destination, which times, with CUDA events:
  masked : tq_partition_push_regions of every source (probe side: LEFT OUTER, keep_misses, a NULL bitmap on the payload
           column so the mask word travels) -> tq_region_gather -> tq_join_put_probe of the gathered rows
  inner  : tq_partition_push_regions of NOT NULL columns -> tq_join_put_probe_segments over the regions in place
on the same data and the same build table (every rank's build shard), and checks every output row of both (B.v = 7 B.k + 1,
B.k = P.k = mix64(P.v) % N_build, as many rows as probe rows).  The receive buffers and the kept miss rows are
tests/exchange_ref.py's Regions, with dist.RegionLayout's argument tables.  Prints one JSON line with the card name and power limit.

    python scripts/region_outer_probe.py [--ranks 2] [--build-rows 12500000] [--probe-rows 125000000] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=2)
    ap.add_argument("--build-rows", type=int, default=12_500_000)
    ap.add_argument("--probe-rows", type=int, default=125_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    import exchange_ref as X
    from tinysql_b200 import _lib as L
    from tinysql_b200 import dist as D
    lib = L.load()
    L.check(lib.tq_init(0))
    dev = torch.device("cuda", 0)
    W, nb, npr = args.ranks, args.build_rows, args.probe_rows
    shards = [D.gen_dist_tables(r, W, nb, npr) for r in range(W)]
    dt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    src = [[dt(x) for x in sh] for sh in shards]                     # bk, bv, pk, pv per source
    del shards
    pv_nn = torch.full(((npr + 63) // 64 * 8 + 8,), 0xFF, dtype=torch.uint8, device=dev)  # a bitmap that says NOT NULL everywhere
    cap = npr                                                        # one destination receives every row of every source
    ptr = lambda t: t.data_ptr()
    torch.cuda.synchronize()
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def alloc(nbytes):
        return torch.empty((nbytes + 7) // 8, dtype=torch.int64, device=dev)

    # the destination's regions: (k, v) for the inner join, (k, v, mask) for the masked one; the kept misses of the sources
    regs = {False: X.Regions(lib, W, 2, cap, guard=0), True: X.Regions(lib, W, 3, cap, guard=0)}
    miss = X.Regions(lib, 1, 3, 64, guard=0)
    g_cols = [alloc(W * cap * 8) for _ in range(2)]
    g_bm = [alloc(((W * cap + 63) // 64) * 8 + 8) for _ in range(2)]
    epoch = [0]

    def build_handle(jt):
        bk = np.concatenate(shards_bk)
        t = (C.c_int32 * 2)(1, 1)
        k = (C.c_int32 * 1)(0)
        desc = L.TQJoinDesc(jt, 0, 2, t, 2, t, 1, k, k, 0, 0)
        h = C.c_void_p()
        L.check(lib.tq_join_create(C.byref(desc), C.byref(h)))
        b = [dt(bk), dt(bk * 7 + 1)]
        L.check(lib.tq_join_put_build(h, D._tq_cols(L, b, len(bk)), L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        return h, b

    shards_bk = [s[0].cpu().numpy() for s in src]

    def drain(h, check):
        out = (L.TQColumn * 4)()
        n, eof = C.c_int64(0), C.c_int32(0)
        rows, ok = 0, True
        while True:
            L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
            if n.value == 0:
                break
            rows += n.value
            if check:
                from tinysql_b200.chunk import device_to_host
                pk, pv, bk, bv = (device_to_host(1, out[c].data, None, n.value).values for c in range(4))
                ok = ok and bool(np.array_equal(bv, bk * 7 + 1) and np.array_equal(bk, pk))
                ok = ok and bool(np.array_equal(pk, (D.mix64_np(pv) % np.uint64(nb * W)).astype(np.int64)))
        return rows, ok

    def run(masked, check=False):
        """every source pushes into the destination's regions, then the receive side; returns (push, gather, join) ms, rows, ok"""
        jt = 1 if masked else 0
        h, keep = build_handle(jt)
        e = [ev() for _ in range(4)]
        reg = regs[masked]
        epoch[0] += 1
        try:
            torch.cuda.synchronize()
            lib.tq_device_synchronize()
            e[0].record()
            for s in range(W):
                pk, pv = src[s][2], src[s][3]
                cols = D._tq_cols(L, [pk, pv], npr)
                dest, cnts = reg.push_tables(0, s)                   # n_parts = 1: destination 0's entries
                md, ms = None, None
                if masked:
                    cols[1].null_bitmap = ptr(pv_nn)
                    md, ms = miss.push_tables(0, 0)[0], miss.slot_ptr(0, 0, 0)
                L.check(lib.tq_partition_push_regions(2, cols, 0, npr, 1, None, int(masked), dest, cnts, cap, md, ms, 64 if masked else 0, s, epoch[0]))
            for s in range(W):
                L.check(lib.tq_partition_push_sync(s))
            e[1].record()
            L.check(reg.wait(0, epoch[0]))
            if masked:
                outc = (L.TQColumn * 2)()
                for c in range(2):
                    outc[c].data, outc[c].null_bitmap = ptr(g_cols[c]), ptr(g_bm[c])
                n = C.c_int64(0)
                L.check(lib.tq_region_gather(W, C.c_void_p(reg.slot_ptr(0, 0, 0)), cap, 2, 1, reg.region_table(0, 0), outc, W * cap, C.byref(n)))
                e[2].record()
                L.check(lib.tq_join_put_probe(h, outc, None, L.TQ_MEM_DEVICE))
            else:
                e[2].record()
                L.check(lib.tq_join_put_probe_segments(h, W, reg.region_table(0, 0), reg.count_ptrs(0, 0), cap))
            L.check(lib.tq_join_probe_eof(h))
            rows, ok = drain(h, check)
            e[3].record()
            torch.cuda.synchronize()
            lib.tq_device_synchronize()
        finally:
            lib.tq_join_destroy(h)
        return [e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3])], rows, ok

    # the W sources push with n_parts = 1 into one destination, which joins every probe row against every build row: the
    # exchange's kernels and the local join at the per-rank C5 shape, without the NVLink transfer one GPU cannot make
    out = {"card": card(), "ranks": W, "build_rows_per_rank": nb, "probe_rows_per_rank": npr}
    for name, masked in (("inner_segmented", False), ("left_outer_masked_gather", True)):
        rows, ok = run(masked, check=True)[1:]
        ok = ok and rows == W * npr
        times = [run(masked)[0] for _ in range(args.reps)]
        med = np.median(np.array(times), axis=0)
        out[name] = {"push_ms": round(float(med[0]), 3), "gather_ms": round(float(med[1]), 3) if masked else None,
                     "join_ms": round(float(med[2]), 3), "rows": int(rows), "rows_checked_ok": ok}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
