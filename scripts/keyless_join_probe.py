"""Throughput of the key-less hash join (tq_join_desc.n_keys == 0), device in, results lent by tq_join_next_device.

  python scripts/keyless_join_probe.py [--legs a,b,c] [--out FILE]

  a  cross join without conditions: build 1e4 x probe 1e5 int64 (k, v) = 1e9 joined rows.  Reports joined rows/s (wall time
     from the first put to the last tq_join_next_device), the materialisation kernel's written bytes/s over its CUDA-event time
     (tq_join_stats[5] per result batch; 4 x 8 B values + 4 NOT-NULL bits per row) as a share of 3.35 TB/s (H100 SXM data
     sheet), and the host time per result batch outside that kernel.
  b  B.v < P.v AND B.v >= P.v - 1000 as a comparison list (the second bound reads a probe column P.w = P.v - 1000) over
     1e5 x 1e5 = 1e10 pairs: pairs evaluated per second and joined rows/s.
  c  the same selectivity as a program with arithmetic, B.v < P.v AND B.v + 1000 >= P.v: pairs/s.
Every leg checks its row count against the closed form.  One JSON line per leg, with the card name and power limit."""
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

from tinysql_b200 import _lib as L  # noqa: E402
from tinysql_b200.chunk import INT64, Column, DeviceColumn  # noqa: E402
from tinysql_b200.expression import Col, Const, Func, JoinProgram  # noqa: E402

HBM_PEAK = 3.35e12   # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def run(lib, nb, npr, bcols, pcols, conds=None, program=None):
    bt, pt = (C.c_int32 * len(bcols))(*[INT64] * len(bcols)), (C.c_int32 * len(pcols))(*[INT64] * len(pcols))
    d = L.TQJoinDesc(0, 0, len(bcols), bt, len(pcols), pt, 0, None, None, 0, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    if conds:
        arr = (L.TQJoinCond * len(conds))(*[L.TQJoinCond(op, a, b, 0, 0) for op, a, b in conds])
        L.check(lib.tq_join_set_other_conditions(h, len(conds), arr))
    if program:
        JoinProgram(program).set_on(lib.tq_join_set_other_program, h)
    db = [DeviceColumn.from_host(Column(INT64, c)) for c in bcols]
    dp = [DeviceColumn.from_host(Column(INT64, c)) for c in pcols]
    L.check(lib.tq_device_synchronize())
    stats = (C.c_int64 * 8)()
    arr = (L.TQColumn * (len(bcols) + len(pcols)))()
    n, eof = C.c_int64(0), C.c_int32(0)
    t0 = time.perf_counter()
    L.check(lib.tq_join_put_build(h, (L.TQColumn * len(db))(*[x.tq() for x in db]), L.TQ_MEM_DEVICE))
    L.check(lib.tq_join_finalize_build(h))
    L.check(lib.tq_join_put_probe(h, (L.TQColumn * len(dp))(*[x.tq() for x in dp]), None, L.TQ_MEM_DEVICE))
    L.check(lib.tq_join_probe_eof(h))
    rows, batches, kern_ns, last = 0, 0, 0, -1
    while True:
        L.check(lib.tq_join_next_device(h, arr, C.byref(n), C.byref(eof)))
        if n.value == 0:
            break
        rows += n.value
        batches += 1
        L.check(lib.tq_join_stats(h, stats))
        if stats[4] != last:   # a batch was built in this call: its materialisation time
            kern_ns += stats[5]
            last = stats[4]
    wall = time.perf_counter() - t0
    lib.tq_join_destroy(h)
    for x in db + dp:
        x.free()
    return rows, batches, wall, kern_ns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="a,b,c")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = L.load()
    L.check(lib.tq_init(0))
    info = card()
    lines = []
    rng = np.random.default_rng(1)
    if "a" in a.legs:
        nb, npr = 10_000, 100_000
        rows, batches, wall, kern_ns = run(lib, nb, npr, [np.arange(nb), rng.integers(0, 1 << 40, nb)], [np.arange(npr), rng.integers(0, 1 << 40, npr)])
        assert rows == nb * npr, rows
        bytes_w = rows * (32 + 0.5)
        lines.append({"leg": "a", "card": info, "rows": rows, "batches": batches, "wall_s": wall, "rows_per_s": rows / wall,
                      "materialize_bytes_per_s": bytes_w / (kern_ns * 1e-9), "share_of_hbm_peak_3.35TBps": bytes_w / (kern_ns * 1e-9) / HBM_PEAK,
                      "host_gap_per_batch_ms": (wall - kern_ns * 1e-9) / batches * 1e3})
    nb = npr = 100_000
    bv = np.arange(nb)
    pv = rng.integers(0, nb + 1000, npr)
    want = int((np.minimum(pv, nb) - np.maximum(pv - 1000, 0)).clip(0).sum())
    if "b" in a.legs:
        rows, batches, wall, _ = run(lib, nb, npr, [bv], [pv, pv - 1000], conds=[(0, 2, 0), (3, 2, 1)])   # B.v < P.v, B.v >= P.w
        assert rows == want, (rows, want)
        lines.append({"leg": "b", "card": info, "pairs": nb * npr, "rows": rows, "wall_s": wall, "pairs_per_s": nb * npr / wall, "rows_per_s": rows / wall})
    if "c" in a.legs:
        prog = [Func("lt", Col(1), Col(0)), Func("ge", Func("plus", Col(1), Const(1000)), Col(0))]
        rows, batches, wall, _ = run(lib, nb, npr, [bv], [pv], program=prog)
        assert rows == want, (rows, want)
        lines.append({"leg": "c", "card": info, "pairs": nb * npr, "rows": rows, "wall_s": wall, "pairs_per_s": nb * npr / wall, "rows_per_s": rows / wall})
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
