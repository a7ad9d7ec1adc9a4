"""Cost of OtherConditions inside the hash join at the C3 shape (1e7 unique build rows x 1e8 probe rows, 8-byte columns,
inputs resident in HBM, every probe row matches once, results lent by tq_join_next_device).

  python scripts/join_cond_probe.py [--lib PATH] [--modes none,cond,prog,arith] [--reps 3]
      one process, one library: wall time of the whole join (create .. last tq_join_next_device, which waits for the device)
      per mode, median of --reps after one warm-up, plus the joined-row count checked against numpy and a sample against
      the CPU oracle.
        none  : no conditions
        cond  : the comparison list  B.v < P.v                 (tq_join_set_other_conditions, ~65 % of the joined rows pass)
        prog  : the same comparison as a program               (tq_join_set_other_program)
        arith : the program  B.v + P.v > 85e6                  (~50 % pass)
  python scripts/join_cond_probe.py --compare PARENT_LIB [--reps 3]
      alternates a library built from the parent commit (comparison list only) with this tree's library, one process per
      run, parent first then branch, --reps times; prints every run and the medians.
  python scripts/join_cond_probe.py --profile [--lib PATH]
      one run per mode under torch.profiler (CUDA activities): device time per kernel, so the condition pass (k_oc_eval,
      k_oc_decide, the scan, k_oc_compact) can be read apart from the probe.

Bytes per joined row of the condition pass (computed from the shapes, 4 output columns, pass fraction s):
  k_oc_eval 2 x 8 B inputs + 1 B flag, k_oc_decide 1 + 4 B, scan 4 + 4 B, k_oc_compact 4 + 1 B + s x (4 B pos + 4 x 8 B read
  + 4 x 8 B write)."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_BUILD, N_PROBE = 10_000_000, 100_000_000
THRESH = 85_000_000


def cond_bytes_per_row(s):
    return 17 + 5 + 8 + 5 + s * (4 + 64)


def load(path):
    """the library at `path` with the bindings of this tree; symbols an older library lacks are left unbound"""
    from tinysql_b200 import _lib as L
    lib = C.CDLL(path)
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = res, args
    L._lib = lib
    L.check(lib.tq_init(0))
    return L, lib


def tables():
    rb, rp = np.random.default_rng(3), np.random.default_rng(4)
    bk = rb.permutation(N_BUILD).astype(np.int64)
    pk = rp.integers(0, N_BUILD, N_PROBE, dtype=np.int64)
    return bk, bk * 7 + 1, pk, np.arange(N_PROBE, dtype=np.int64)


def program(mode):
    from tinysql_b200.expression import Col, Const, Func
    # output = B.k B.v P.k P.v (the build side is the left child)
    if mode == "prog":
        return [Func("lt", Col(1), Col(3))]
    return [Func("gt", Func("plus", Col(1), Col(3)), Const(THRESH))]


def join_once(L, lib, d_b, d_p, mode):
    from tinysql_b200.expression import JoinProgram
    t, k = (C.c_int32 * 2)(1, 1), (C.c_int32 * 1)(0)
    h = C.c_void_p()
    t0 = time.perf_counter()
    L.check(lib.tq_join_create(C.byref(L.TQJoinDesc(0, 1, 2, t, 2, t, 1, k, k, 0, 0)), C.byref(h)))
    if mode == "cond":
        L.check(lib.tq_join_set_other_conditions(h, 1, (L.TQJoinCond * 1)(L.TQJoinCond(0, 1, 3, 0, 0))))
    elif mode in ("prog", "arith"):
        JoinProgram(program(mode)).set_on(lib.tq_join_set_other_program, h)
    L.check(lib.tq_join_put_build(h, (L.TQColumn * 2)(*[c.tq() for c in d_b]), L.TQ_MEM_DEVICE))
    L.check(lib.tq_join_finalize_build(h))
    L.check(lib.tq_join_put_probe(h, (L.TQColumn * 2)(*[c.tq() for c in d_p]), None, L.TQ_MEM_DEVICE))
    L.check(lib.tq_join_probe_eof(h))
    rows = 0
    while True:
        out, n, eof = (L.TQColumn * 4)(), C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
        rows += n.value
        if n.value == 0 and eof.value:
            break
    L.check(lib.tq_device_synchronize())
    sec = time.perf_counter() - t0
    lib.tq_join_destroy(h)
    return sec, rows


def sample_check(L, lib, bk, bv, pk, pv, mode):
    """the library and the CPU oracle on the full build side and a 200k-row probe sample"""
    import oracle_py as O
    from join_program_oracle import join_with_program
    from tinysql_b200.chunk import INT64, Column
    from tinysql_b200.executor import HashJoinExec, MockDataSource
    from util import assert_same_multiset
    sel = np.random.default_rng(9).choice(N_PROBE, 200_000, replace=False)
    b, p = [Column(INT64, bk), Column(INT64, bv)], [Column(INT64, pk[sel]), Column(INT64, pv[sel])]
    conds = [(0, 1, 3)] if mode == "cond" else ()
    prog = program(mode) if mode in ("prog", "arith") else ()
    e = HashJoinExec(MockDataSource([INT64, INT64], p, 1 << 20), MockDataSource([INT64, INT64], b, 1 << 20), [0], [0], 0, True,
                     other_conditions=conds, other_program=prog)
    e.Open()
    got = e.drain()
    e.Close()
    if prog:
        want, _ = join_with_program("hash", 0, True, [INT64, INT64], b, [INT64, INT64], p, [0], [0], prog)
    else:
        want = O.hash_join(0, True, [INT64, INT64], b, [INT64, INT64], p, [0], [0], None, conds)
    assert_same_multiset(got, want)
    return got.num_rows()


def expected_rows(bv, pk, pv, mode):
    bvp = pk * 7 + 1   # B.v of the build row each probe row matches
    if mode == "none":
        return N_PROBE
    if mode in ("cond", "prog"):
        return int(np.count_nonzero(bvp < pv))
    return int(np.count_nonzero(bvp + pv > THRESH))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run_modes(path, modes, reps):
    from tinysql_b200.chunk import INT64, Column, DeviceColumn
    L, lib = load(path)
    bk, bv, pk, pv = tables()
    d_b = [DeviceColumn(INT64, N_BUILD, with_bitmap=False), DeviceColumn(INT64, N_BUILD, with_bitmap=False)]
    d_p = [DeviceColumn(INT64, N_PROBE, with_bitmap=False), DeviceColumn(INT64, N_PROBE, with_bitmap=False)]
    for d, a in zip(d_b + d_p, (bk, bv, pk, pv)):
        L.check(lib.tq_memcpy_h2d(d._data, a.ctypes.data, a.nbytes))
    res = {"lib": path, "gpu": gpu_info(), "modes": {}}
    for mode in modes:
        join_once(L, lib, d_b, d_p, mode)   # warm-up
        times, rows = [], 0
        for _ in range(reps):
            sec, rows = join_once(L, lib, d_b, d_p, mode)
            times.append(sec)
        want = expected_rows(bv, pk, pv, mode)
        r = {"join_ms": [round(x * 1e3, 2) for x in times], "median_ms": round(statistics.median(times) * 1e3, 2), "rows": rows,
             "rows_ok": rows == want}
        if mode != "none":
            s = want / N_PROBE
            r["pass_fraction"] = round(s, 4)
            r["cond_pass_bytes_per_joined_row"] = cond_bytes_per_row(s)
            if mode != "cond" or hasattr(lib, "tq_join_set_other_program"):
                r["sample_rows_match_oracle"] = sample_check(L, lib, bk, bv, pk, pv, mode)
        res["modes"][mode] = r
    for d in d_b + d_p:
        d.free()
    return res


def profile(path, modes):
    import torch
    from torch.profiler import ProfilerActivity
    from tinysql_b200.chunk import INT64, DeviceColumn
    L, lib = load(path)
    bk, bv, pk, pv = tables()
    d_b = [DeviceColumn(INT64, N_BUILD, with_bitmap=False), DeviceColumn(INT64, N_BUILD, with_bitmap=False)]
    d_p = [DeviceColumn(INT64, N_PROBE, with_bitmap=False), DeviceColumn(INT64, N_PROBE, with_bitmap=False)]
    for d, a in zip(d_b + d_p, (bk, bv, pk, pv)):
        L.check(lib.tq_memcpy_h2d(d._data, a.ctypes.data, a.nbytes))
    out = {"lib": path, "gpu": gpu_info(), "modes": {}}
    for mode in modes:
        join_once(L, lib, d_b, d_p, mode)
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            join_once(L, lib, d_b, d_p, mode)
        per = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                nm = ev.name if len(ev.name) < 80 else ev.name[:80]
                a = per.setdefault(nm, [0, 0.0])
                a[0] += 1
                a[1] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
        top = sorted(per.items(), key=lambda kv: -kv[1][1])[:14]
        oc = sum(v[1] for k, v in per.items() if "k_oc_" in k)
        out["modes"][mode] = {"k_oc_ms": round(oc, 3), "kernels": [(k, v[0], round(v[1], 3)) for k, v in top]}
    for d in d_b + d_p:
        d.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "tinysql_b200", "lib", "libtinysql_b200.so"))
    ap.add_argument("--modes", default="none,cond,prog,arith")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--compare", default=None, help="library built from the parent commit")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if a.profile:
        print(json.dumps({"join_cond_profile": profile(a.lib, a.modes.split(","))}))
        return
    if not a.compare:
        print(json.dumps({"join_cond_probe": run_modes(a.lib, a.modes.split(","), a.reps)}))
        return
    runs = []
    for _ in range(a.reps):
        for tag, lib, modes in (("parent", a.compare, "none,cond"), ("branch", a.lib, a.modes)):
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--lib", lib, "--modes", modes, "--reps", "3"], capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stderr)
                raise SystemExit(f"{tag} run failed")
            r = json.loads(p.stdout.strip().splitlines()[-1])["join_cond_probe"]
            r["tag"] = tag
            runs.append(r)
            print(json.dumps(r), flush=True)
    summary = {}
    for tag in ("parent", "branch"):
        for mode in a.modes.split(","):
            v = [r["modes"][mode]["median_ms"] for r in runs if r["tag"] == tag and mode in r["modes"]]
            if v:
                summary[f"{tag}_{mode}_ms"] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
    print(json.dumps({"join_cond_compare": summary, "gpu": runs[0]["gpu"]}))


if __name__ == "__main__":
    main()
