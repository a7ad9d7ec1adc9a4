"""The streaming build when one scatter bin holds several sub-tables: a build side large enough that the partition bits plus
the sub-table bits pass the scatter's 9 bits, so each k_build_cluster cluster builds its bin's sub-tables one after another.
Checked with the C3 properties (every probe row joined exactly once, B.v = 7 * B.k + 1) rather than the CPU oracle."""
import ctypes as C

import numpy as np
import pytest

from bench import gen_join_tables, verify_join_result
from tinysql_b200 import _lib as L
from tinysql_b200.chunk import INT64, Column, DeviceColumn

pytestmark = pytest.mark.gpu


def test_stream_build_several_subtables_per_bin(lib, monkeypatch):
    # 3e7 build rows at 20000 rows per partition: the streaming build caps the partitions at 512 (~58.6 K rows each, 4
    # sub-tables each -> 2^11 sub-tables over 2^9 scatter bins); the general build would make 2048 partitions
    monkeypatch.setenv("TQ_JOIN_PART_ROWS", "20000")
    n_build, n_probe = 30_000_000, 30_000_000
    bk, bv, pk, pv = gen_join_tables(n_build, n_probe, n_build)
    d_b = [DeviceColumn.from_host(Column(INT64, bk)), DeviceColumn.from_host(Column(INT64, bv))]
    d_p = [DeviceColumn.from_host(Column(INT64, pk)), DeviceColumn.from_host(Column(INT64, pv))]
    t = (C.c_int32 * 2)(1, 1)
    k = (C.c_int32 * 1)(0)
    d = L.TQJoinDesc(0, 1, 2, t, 2, t, 1, k, k, 0, 0)
    h = C.c_void_p()
    L.check(lib.tq_join_create(C.byref(d), C.byref(h)))
    try:
        barr = (L.TQColumn * 2)(d_b[0].tq(), d_b[1].tq())
        parr = (L.TQColumn * 2)(d_p[0].tq(), d_p[1].tq())
        for a in (barr, parr):
            for i in range(2):
                a[i].null_bitmap = None
        L.check(lib.tq_join_put_build(h, barr, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_finalize_build(h))
        st = (C.c_int64 * 8)()
        L.check(lib.tq_join_stats(h, st))
        assert st[2] == 512, "the streaming build (512 partitions) was not taken"
        L.check(lib.tq_join_put_probe(h, parr, None, L.TQ_MEM_DEVICE))
        L.check(lib.tq_join_probe_eof(h))
        out = (L.TQColumn * 4)()
        n, eof = C.c_int64(0), C.c_int32(0)
        L.check(lib.tq_join_next_device(h, out, C.byref(n), C.byref(eof)))
        rows = n.value
        cols = []
        for c in range(4):
            a = np.empty(rows, dtype=np.int64)
            L.check(lib.tq_memcpy_d2h(a.ctypes.data, out[c].data, rows * 8))
            cols.append(a)
    finally:
        L.check(lib.tq_join_destroy(h))
    res = verify_join_result(rows, cols, pk, n_probe)
    assert res["ok"], res["checks"]
