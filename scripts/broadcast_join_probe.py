"""Cost of dist.BroadcastJoin on ONE GPU with W = 2 emulated ranks (every receive buffer in this GPU's memory, so nothing
crosses NVLink: the NVLink time and the crossover between broadcast and shuffle are not measured here).  Per phase, host
times around calls that end in a synchronise, summed over the ranks, mean over --reps after one warm-up step:
  push           both ranks' tq_partition_push_broadcast, then tq_partition_push_sync
  wait + build   tq_region_wait, the host slot read, tq_join_put_build per source
  finalize       tq_join_finalize_build
  probe + drain  tq_join_put_probe of the local shard, tq_join_probe_eof, tq_join_next_device until empty
and the bytes one rank pushes (W copies of its shard, one of them local).  Workloads:
  (a) c1       BIGINT + VARSTRING keys (5- and 6-byte cells), 1e5 x 1e5 rows per rank, inner join, every probe row matching once
  (b) dim      1e6 build x 1.25e8 probe rows per rank, one INT64 key + payload, inner, NOT NULL; beside it the shuffle's calls
               on the same inputs (dist.RegionJoin's NOT NULL inner path with one probe chunk: tq_partition_push_regions of
               both sides, then per rank the build regions as build chunks and tq_join_put_probe_segments)
  (c) keyless  key-less inner join ON b.x < p.x, 2e3 build x 1e5 probe rows per rank
Row counts are checked against what the inputs imply.  Prints one JSON line with the card name and power limit.

    python scripts/broadcast_join_probe.py [--reps 3] [--probe-rows 125000000]
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
W = 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--probe-rows", type=int, default=125_000_000)
    args = ap.parse_args()
    import torch

    import broadcast_ref as B
    import exchange_ref as X
    from tinysql_b200 import _lib as L
    from tinysql_b200.chunk import BYTES, INT64, Column, DeviceColumn
    from tinysql_b200.dist import RawCol
    lib = L.load()
    L.check(lib.tq_init(0))
    dev = torch.device("cuda", 0)

    def broadcast(name, bt, pt, bcols, pcols, expect_rows, **kw):
        """bcols / pcols: per rank device columns; returns the phase record"""
        nb = max(int(getattr(c[0], "length", 0) or c[0].numel()) for c in bcols)
        em = B.Emulated(lib, W, nb, bt, pt, **kw)
        ph = {"push": [], "wait + build puts": [], "finalize": [], "probe + drain": []}
        try:
            for rep in range(args.reps + 1):
                em.ex.next_epoch()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for r in range(W):
                    em.joins[r].push(bcols[r])
                for r in range(W):
                    L.check(lib.tq_partition_push_sync(r))
                t_push = (time.perf_counter() - t0) * 1e3
                sums, rows = {}, 0
                for r in range(W):
                    n, _, _ = em.joins[r].join(pcols[r])
                    rows += n
                    for k, v in em.joins[r].last_phase.items():
                        sums[k] = sums.get(k, 0.0) + v
                assert rows == expect_rows, (name, rows, expect_rows)
                if rep:
                    ph["push"].append(t_push)
                    for k, v in sums.items():
                        ph[k].append(v)
        finally:
            em.free()
        return {k: round(float(np.mean(v)), 3) for k, v in ph.items()}

    def pushed_bytes(cols_host_bytes):
        return W * cols_host_bytes

    out = {"card": card(), "ranks_emulated": W, "reps": args.reps,
           "note": "emulated ranks on one GPU: every push lands in local HBM; NVLink time and the broadcast/shuffle crossover not measured"}
    rng = np.random.default_rng(1)

    # ---- (a) C1 shape: BIGINT + VARSTRING keys, 1e5 x 1e5 per rank
    n = 100_000
    # the string key is the decimal of the integer key: probe keys 0..n-1 each match rank 0's build row of that key once
    skey = lambda ks: Column(BYTES, [b"%05d" % v for v in ks])
    host_b = [[Column(INT64, ks), skey(ks)] for ks in (rng.permutation(n) + r * n for r in range(W))]
    host_p = [[Column(INT64, ks), skey(ks)] for ks in (rng.permutation(n) for r in range(W))]
    expect = W * n
    db = [[DeviceColumn.from_host(c) for c in cols] for cols in host_b]
    dp = [[DeviceColumn.from_host(c) for c in cols] for cols in host_p]
    out["c1"] = {"build_rows_per_rank": n, "probe_rows_per_rank": n, "rows": expect,
                 "bytes_pushed_per_rank": pushed_bytes(n * 8 + (n + 1) * 8 + n * 6),
                 "phase_ms_sum_over_ranks": broadcast("c1", [INT64, BYTES], [INT64, BYTES], db, dp, expect, build_keys=[0, 1], probe_keys=[0, 1],
                                                      byte_caps=[None, n * 6])}
    for cols in db + dp:
        for c in cols:
            c.free()

    # ---- (b) dimension join: 1e6 build x probe-rows per rank, inner, NOT NULL
    nb, npr = 1_000_000, args.probe_rows
    bk = [torch.randperm(nb, device=dev, dtype=torch.int64) * W + r for r in range(W)]
    bv = [k * 7 + 1 for k in bk]
    pk = [torch.randint(0, nb * W, (npr,), device=dev, dtype=torch.int64) for _ in range(W)]
    pv = [torch.arange(npr, device=dev, dtype=torch.int64) + r * npr for r in range(W)]
    torch.cuda.synchronize()
    out["dim"] = {"build_rows_per_rank": nb, "probe_rows_per_rank": npr, "rows": W * npr, "bytes_pushed_per_rank": pushed_bytes(nb * 16),
                  "broadcast_phase_ms_sum_over_ranks": broadcast("dim", [INT64, INT64], [INT64, INT64], [[bk[r], bv[r]] for r in range(W)],
                                                                 [[pk[r], pv[r]] for r in range(W)], W * npr, build_keys=[0], probe_keys=[0])}
    # the shuffle's calls on the same inputs (RegionJoin's NOT NULL inner path, one probe chunk)
    capb, capp = int(nb / W * 1.25) + (1 << 14), int(npr / W * 1.25) + (1 << 14)
    rb, rp = X.Regions(lib, W, 2, capb, 0), X.Regions(lib, W, 2, capp, 0)
    ph = {"push": [], "wait + build puts": [], "finalize": [], "probe + drain": []}
    t_b, t_p = (C.c_int32 * 2)(1, 1), (C.c_int32 * 2)(1, 1)
    k = (C.c_int32 * 1)(0)
    try:
        for rep in range(args.reps + 1):
            epoch = rep + 1
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for s in range(W):
                L.check(rb.push(s, [bk[s].data_ptr(), bv[s].data_ptr()], nb, s, epoch))
                L.check(rp.push(s, [pk[s].data_ptr(), pv[s].data_ptr()], npr, W + s, epoch))
            for s in range(2 * W):
                L.check(lib.tq_partition_push_sync(s))
            t_push = (time.perf_counter() - t0) * 1e3
            sums, rows = {k2: 0.0 for k2 in ph if k2 != "push"}, 0
            for d in range(W):
                t0 = time.perf_counter()
                d_ = L.TQJoinDesc(0, 1, 2, t_b, 2, t_p, 1, k, k, 0, 0)
                h = C.c_void_p()
                L.check(lib.tq_join_create(C.byref(d_), C.byref(h)))
                try:
                    L.check(rb.wait(d, epoch))
                    L.check(rp.wait(d, epoch))
                    cnt = rb.counts(d)[0]
                    for g in range(W):
                        cols = [RawCol(rb.region_ptr(d, 0, g, c), cnt[g]) for c in range(2)]
                        arr = (L.TQColumn * 2)()
                        for c in range(2):
                            arr[c].length, arr[c].data = cnt[g], cols[c].ptr
                        L.check(lib.tq_join_put_build(h, arr, L.TQ_MEM_DEVICE))
                    L.check(lib.tq_compute_synchronize())
                    t1 = time.perf_counter()
                    L.check(lib.tq_join_finalize_build(h))
                    L.check(lib.tq_compute_synchronize())
                    t2 = time.perf_counter()
                    L.check(lib.tq_join_put_probe_segments(h, W, rp.region_table(d, 0), rp.count_ptrs(d, 0), rp.cap[0]))
                    L.check(lib.tq_join_probe_eof(h))
                    o = (L.TQColumn * 4)()
                    n_, eof = C.c_int64(0), C.c_int32(0)
                    while True:
                        L.check(lib.tq_join_next_device(h, o, C.byref(n_), C.byref(eof)))
                        if n_.value == 0:
                            break
                        rows += n_.value
                    L.check(lib.tq_compute_synchronize())
                    t3 = time.perf_counter()
                finally:
                    lib.tq_join_destroy(h)
                sums["wait + build puts"] += (t1 - t0) * 1e3
                sums["finalize"] += (t2 - t1) * 1e3
                sums["probe + drain"] += (t3 - t2) * 1e3
            assert rows == W * npr, ("shuffle", rows)
            if rep:
                ph["push"].append(t_push)
                for k2, v in sums.items():
                    ph[k2].append(v)
    finally:
        rb.free()
        rp.free()
    out["dim"]["shuffle_bytes_pushed_per_rank"] = (nb + npr) * 16
    out["dim"]["shuffle_phase_ms_sum_over_ranks"] = {k2: round(float(np.mean(v)), 3) for k2, v in ph.items()}
    del bk, bv, pk, pv
    torch.cuda.empty_cache()

    # ---- (c) key-less ON b.x < p.x
    nb, npr = 2_000, 100_000
    kb = [torch.randint(0, 1000, (nb,), device=dev, dtype=torch.int64) for _ in range(W)]
    kp = [torch.randint(0, 1000, (npr,), device=dev, dtype=torch.int64) for _ in range(W)]
    kbh, kph = np.concatenate([x.cpu().numpy() for x in kb]), [x.cpu().numpy() for x in kp]
    srt = np.sort(kbh)
    expect = int(sum(np.searchsorted(srt, p, side="left").sum() for p in kph))
    out["keyless"] = {"build_rows_per_rank": nb, "probe_rows_per_rank": npr, "rows": expect, "bytes_pushed_per_rank": pushed_bytes(nb * 8),
                      "phase_ms_sum_over_ranks": broadcast("keyless", [INT64], [INT64], [[x] for x in kb], [[x] for x in kp], expect,
                                                           outer_is_right=False, other_conditions=[(0, 1, 0)])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
