"""Throughput of the device sort / merge join on the GPU: rows/s of the sort phase (CUDA events inside
tq_sort_eof, tq_sort_stats) for a few key shapes, and wall-clock of the whole operators through the C-ABI with host chunks."""
import ctypes as C
import json
import sys
import time

import numpy as np

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import FLOAT64, INT64, Column, tq_array

lib = L.load()
L.check(lib.tq_init(0))


def sort_once(cols, types, by, n):
    h = C.c_void_p()
    d = L.TQSortDesc(len(types), (C.c_int32 * len(types))(*types), len(by), (C.c_int32 * len(by))(*[c for c, _ in by]),
                     (C.c_int32 * len(by))(*[1 if x else 0 for _, x in by]), 0, -1)
    L.check(lib.tq_sort_create(C.byref(d), C.byref(h)))
    t0 = time.perf_counter()
    L.check(lib.tq_sort_put(h, tq_array(cols), L.TQ_MEM_HOST))
    L.check(lib.tq_sort_eof(h))
    t1 = time.perf_counter()
    st = (C.c_int64 * 4)()
    lib.tq_sort_stats(h, st)
    out = [Column.empty(t, 1024) for t in types]
    nr, eof = C.c_int64(0), C.c_int32(0)
    L.check(lib.tq_sort_next(h, 1024, tq_array(out, 1024), C.byref(nr), C.byref(eof)))
    first = [c.values[: nr.value].copy() for c in out]
    lib.tq_sort_destroy(h)
    return st[1] * 1e-9, int(st[3]), int(st[2]), t1 - t0, first


res = []
rng = np.random.default_rng(1)
n = 50_000_000
rid = Column(INT64, np.arange(n))
for name, key in (("int64 uniform in [0, 1e6): 3 digit passes", Column(INT64, rng.integers(0, 1_000_000, n))),
                  ("int64 full range: 8 digit passes", Column(INT64, rng.integers(-(1 << 62), 1 << 62, n))),
                  ("float64 uniform [0, 1)", Column(FLOAT64, rng.random(n)))):
    types = [key.tp, INT64]
    sort_once([key, rid], types, [(0, False)], n)   # warm-up (allocations)
    sec, passes, launches, wall, first = sort_once([key, rid], types, [(0, False)], n)
    ok = bool(np.all(np.diff(first[0]) >= 0)) and bool(np.array_equal(first[0], key.values[first[1]]))
    # per pass: count reads 8 B/row; scatter reads 12 and writes 12 B/row; + one key gather (12 B read + 8 B write + the column gather)
    res.append({"case": name, "rows": n, "sort_phase_ms": sec * 1e3, "rows_per_s": n / sec, "radix_passes": passes, "launches": launches,
                "approx_GBps": (passes * 32 + 28) * n / sec / 1e9, "eof_wall_s_incl_upload_and_result_copy": wall, "first_chunk_ordered": ok})
print(json.dumps({"sort_probe": res}))
