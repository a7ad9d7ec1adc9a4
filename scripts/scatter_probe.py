"""Times the calls that go through the radix scatters of join.cu, at user sizes, and checks what they compute.

  python scripts/scatter_probe.py [--lib PATH] [--cases outer_fast,outer_nullable,push8,agg_part,stream_build] [--reps 5]
      one process, one library: wall time per case (host clock around calls that end in a device synchronise), median of
      --reps after one warm-up, plus a row count and a checksum of every result column (64-bit wrapping sum of the bits, so
      the order the scatter leaves rows in does not matter).
        outer_fast      LEFT OUTER hash join, 1e7 unique build rows x 5e7 probe rows, 2 + 2 NOT NULL INT64 columns: the
                        general partitioned probe, scattered by k_probe_scatter_fast
        outer_nullable  the same join with nullable probe columns (no NULL in them): k_probe_scatter
        push8           tq_partition_push_regions of 2e7 rows x 4 NOT NULL columns into 8 regions on this GPU, caps from the
                        host-side destinations: k_probe_scatter_fast<4>
        agg_part        GROUP BY of 8e6 rows into ~1.5e6 groups (SUM, COUNT, FIRSTROW over INT64): the HashAgg pre-aggregation
                        at 2^10 partitions, scattered by scatter_rows_by_hash (k_probe_scatter_fast); time = tq_agg_stats[2]
        stream_build    inner PK-FK hash join, 1e7 unique build rows x 2e7 probe rows: the streaming build (k_scatter_aos)
                        and the positional probe (k_scatter_cols); time = the whole join
  python scripts/scatter_probe.py --compare PARENT_LIB [--reps 3]
      alternates a library built from the parent commit with this tree's library, one process per run, parent first, --reps
      times each; prints every run, the medians per case and whether rows and checksums agree between the two libraries.
      A library from before the region push had one entry point exports it, with the same arguments, under its former
      name: tq_partition_push_regions with the suffix _masked.  Such a library is called through that name."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = "outer_fast,outer_nullable,push8,agg_part,stream_build"


def load(path):
    """the library at `path` with the bindings of this tree"""
    from tinysql_b200 import _lib as L
    lib = C.CDLL(path)
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = res, args
    push = "tq_partition_push_regions"
    former = getattr(lib, f"{push}_masked", None)      # the same push of a library from before it had one entry point
    if former is not None:
        former.restype, former.argtypes = L.SYMBOLS[push]
        setattr(lib, push, former)
    L._lib = lib
    L.check(lib.tq_init(0))
    return L, lib


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def dev_col(L, lib, a, nullable=False):
    from tinysql_b200.chunk import INT64, DeviceColumn
    d = DeviceColumn(INT64, len(a), with_bitmap=nullable)
    L.check(lib.tq_memcpy_h2d(d._data, a.ctypes.data, a.nbytes))
    if nullable:
        L.check(lib.tq_memset_device(d._bm, 0xFF, d.bm_bytes))
    return d


def col_sum(L, lib, ptr, n):
    h = np.empty(n, dtype=np.uint64)
    if n:
        L.check(lib.tq_memcpy_d2h(h.ctypes.data, ptr, n * 8))
    return int(h.sum(dtype=np.uint64))


def run_join(L, lib, d_b, d_p, join_type, check):
    """one hash join of the resident columns: (seconds, rows, checksums, build path)"""
    t, k = (C.c_int32 * 2)(1, 1), (C.c_int32 * 1)(0)
    h = C.c_void_p()
    t0 = time.perf_counter()
    L.check(lib.tq_join_create(C.byref(L.TQJoinDesc(join_type, 0 if join_type else 1, 2, t, 2, t, 1, k, k, 0, 0)), C.byref(h)))
    L.check(lib.tq_join_put_build(h, (L.TQColumn * 2)(*[c.tq() for c in d_b]), L.TQ_MEM_DEVICE))
    L.check(lib.tq_join_finalize_build(h))
    L.check(lib.tq_join_put_probe(h, (L.TQColumn * 2)(*[c.tq() for c in d_p]), None, L.TQ_MEM_DEVICE))
    L.check(lib.tq_join_probe_eof(h))
    rows, sums = 0, [0, 0, 0, 0]
    while True:
        out, n, eof = (L.TQColumn * 4)(), C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
        rows += n.value
        if check and n.value:
            for c in range(4):
                sums[c] = (sums[c] + col_sum(L, lib, out[c].data, n.value)) & (2**64 - 1)
        if n.value == 0 and eof.value:
            break
    L.check(lib.tq_device_synchronize())
    sec = time.perf_counter() - t0
    path = C.c_int32(-1)
    L.check(lib.tq_join_build_path(h, C.byref(path)))
    lib.tq_join_destroy(h)
    return sec, rows, sums, path.value


def case_join(L, lib, reps, join_type, n_build, n_probe, nullable):
    rb, rp = np.random.default_rng(3), np.random.default_rng(4)
    bk = rb.permutation(n_build).astype(np.int64)
    pk = rp.integers(0, n_build, n_probe, dtype=np.int64)
    d_b = [dev_col(L, lib, bk), dev_col(L, lib, bk * 7 + 1)]
    d_p = [dev_col(L, lib, pk, nullable), dev_col(L, lib, np.arange(n_probe, dtype=np.int64), nullable)]
    _, rows, sums, path = run_join(L, lib, d_b, d_p, join_type, True)
    times = [run_join(L, lib, d_b, d_p, join_type, False)[0] for _ in range(reps)]
    for d in d_b + d_p:
        d.free()
    return times, {"rows": rows, "checksums": [str(s) for s in sums], "build_path": path}


def case_push8(L, lib, reps):
    from tinysql_b200.chunk import INT64, DeviceColumn
    from tinysql_b200.dist import dest_rank_np
    n, ncols, n_parts = 20_000_000, 4, 8
    rng = np.random.default_rng(7)
    cols = [rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64)] + [np.arange(n, dtype=np.int64) * (c + 3) + c for c in range(1, ncols)]
    d_in = [dev_col(L, lib, a) for a in cols]
    tq = (L.TQColumn * ncols)(*[d.tq() for d in d_in])
    for c in range(ncols):
        tq[c].null_bitmap = None
    counts = np.bincount(dest_rank_np(cols[0], n_parts), minlength=n_parts)
    cap = int(counts.max())
    dst = [[DeviceColumn(INT64, cap, with_bitmap=False) for _ in range(ncols)] for q in range(n_parts)]
    slots = DeviceColumn(INT64, 2 * n_parts, with_bitmap=False)
    ptrs = (C.c_void_p * (n_parts * ncols))(*[d._data.value for dq in dst for d in dq])
    cnts = (C.c_void_p * n_parts)(*[slots._data.value + 16 * q for q in range(n_parts)])

    def once():
        t0 = time.perf_counter()
        L.check(lib.tq_partition_push_regions(ncols, tq, 0, n, n_parts, None, 0, ptrs, cnts, cap, None, None, 0, 0, 1))
        L.check(lib.tq_partition_push_sync(0))
        return time.perf_counter() - t0

    once()
    pub = np.zeros(2 * n_parts, np.uint64)
    L.check(lib.tq_memcpy_d2h(pub.ctypes.data, slots._data, pub.nbytes))
    rows = [int(r) for r in pub[0::2]]
    if rows != [int(c) for c in counts]:
        raise SystemExit(f"push8: published rows {rows}, host destinations {list(counts)}")
    sums = [str(col_sum(L, lib, d._data, rows[q])) for q, dq in enumerate(dst) for d in dq]
    times = [once() for _ in range(reps)]
    for d in d_in + [d for dq in dst for d in dq] + [slots]:
        d.free()
    return times, {"rows": sum(rows), "counts": rows, "checksums": sums}


def case_agg(L, lib, reps):
    from tinysql_b200.chunk import INT64
    n, groups = 8_000_000, 1_500_000
    k = np.random.default_rng(5).integers(0, groups, n, dtype=np.int64)
    x = np.random.default_rng(6).integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    dk, dx = dev_col(L, lib, k), dev_col(L, lib, x)
    types = (C.c_int32 * 2)(INT64 | 0x100, INT64 | 0x100)
    gb = (C.c_int32 * 1)(0)
    funcs = (L.TQAggFunc * 3)(L.TQAggFunc(1, 1), L.TQAggFunc(0, -1), L.TQAggFunc(5, 0))
    desc = L.TQAggDesc(2, types, 1, gb, 3, funcs, groups)

    def once(check):
        h = C.c_void_p()
        L.check(lib.tq_agg_create(C.byref(desc), C.byref(h)))
        cols = (L.TQColumn * 2)(dk.tq(), dx.tq())
        L.check(lib.tq_agg_put(h, cols, L.TQ_MEM_DEVICE))
        L.check(lib.tq_agg_eof(h))
        st = (C.c_int64 * 4)()
        lib.tq_agg_stats(h, st)
        rows, sums = 0, [0, 0, 0]
        if check:
            while True:
                out, m, eof = (L.TQColumn * 3)(), C.c_int64(0), C.c_int32(0)
                L.check(lib.tq_agg_next_device(h, out, C.byref(m), C.byref(eof)))
                rows += m.value
                for c in range(3):
                    if m.value:
                        sums[c] = (sums[c] + col_sum(L, lib, out[c].data, m.value)) & (2**64 - 1)
                if m.value == 0 or eof.value:
                    break
        L.check(lib.tq_agg_destroy(h))
        return st[2] / 1e9, rows, sums

    _, rows, sums = once(True)
    times = [once(False)[0] for _ in range(reps)]
    dk.free()
    dx.free()
    return times, {"rows": rows, "checksums": [str(s) for s in sums]}


def run_cases(path, cases, reps):
    L, lib = load(path)
    res = {"lib": path, "gpu": gpu_info(), "cases": {}}
    for case in cases:
        if case == "outer_fast":
            times, chk = case_join(L, lib, reps, 1, 10_000_000, 50_000_000, False)
        elif case == "outer_nullable":
            times, chk = case_join(L, lib, reps, 1, 10_000_000, 50_000_000, True)
        elif case == "stream_build":
            times, chk = case_join(L, lib, reps, 0, 10_000_000, 20_000_000, False)
        elif case == "push8":
            times, chk = case_push8(L, lib, reps)
        elif case == "agg_part":
            times, chk = case_agg(L, lib, reps)
        else:
            raise SystemExit(f"unknown case {case}")
        res["cases"][case] = {"ms": [round(t * 1e3, 3) for t in times], "median_ms": round(statistics.median(times) * 1e3, 3), **chk}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "tinysql_b200", "lib", "libtinysql_b200.so"))
    ap.add_argument("--cases", default=CASES)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--compare", default=None, help="library built from the parent commit")
    a = ap.parse_args()
    cases = a.cases.split(",")
    if not a.compare:
        print(json.dumps({"scatter_probe": run_cases(a.lib, cases, a.reps)}))
        return
    runs = []
    for _ in range(a.reps):
        for tag, lib in (("parent", a.compare), ("branch", a.lib)):
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--lib", lib, "--cases", a.cases, "--reps", "5"], capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stderr)
                raise SystemExit(f"{tag} run failed")
            r = json.loads(p.stdout.strip().splitlines()[-1])["scatter_probe"]
            r["tag"] = tag
            runs.append(r)
            print(json.dumps(r), flush=True)
    summary, same = {}, {}
    for case in cases:
        for tag in ("parent", "branch"):
            v = [r["cases"][case]["median_ms"] for r in runs if r["tag"] == tag]
            summary[f"{tag}_{case}_ms"] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
        results = {json.dumps({k: v for k, v in r["cases"][case].items() if k not in ("ms", "median_ms")}, sort_keys=True) for r in runs}
        same[case] = len(results) == 1
    print(json.dumps({"scatter_compare": summary, "results_agree": same, "gpu": runs[0]["gpu"]}))


if __name__ == "__main__":
    main()
