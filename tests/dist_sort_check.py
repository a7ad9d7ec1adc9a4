"""torchrun entry: dist.RegionSort across real GPUs — ORDER BY a nullable VARCHAR DESC then a BIGINT, with a DOUBLE payload,
over two steps that reuse the regions, then ORDER BY ... LIMIT with a window that spans ranks — against sort_ref over the
gathered shards in rank order.  Launched by tests/test_gpu_dist_sort.py (2 ranks when 2 GPUs are visible, one rank otherwise)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    import region_sort_ref as RS
    import sort_ref as SR
    from tinysql_b200 import _lib as L
    from tinysql_b200 import dist as D
    from tinysql_b200.chunk import BYTES, Column, VarColumn
    lib = L.load()
    L.check(lib.tq_init(local))
    I64, F64 = L.TQ_TYPE_INT64, L.TQ_TYPE_FLOAT64

    rng = np.random.default_rng(500 + rank)
    n = 100_000
    words = [b""] + [b"key-%05d" % i for i in range(3000)]
    s = VarColumn(BYTES, [None if rng.random() < 0.02 else words[i] for i in rng.integers(0, len(words), n)])
    k = Column(I64, rng.integers(-50, 50, n).astype(np.int64), rng.random(n) >= 0.05)
    x = Column(F64, rng.random(n))
    types, by = [BYTES, I64, F64], [(0, True), (1, False)]
    caps = [None] * world
    dist.all_gather_object(caps, int(s.offsets[-1]) + 1)
    byte_caps = [max(caps), None, None]                  # every rank passes the same numbers: the layout is shared
    shard = [s, k, x]
    gathered = [None] * world
    dist.all_gather_object(gathered, [c.tolist() for c in shard])
    full = [r for g in gathered for r in zip(*g)]
    dev = RS.device(shard)
    torch.cuda.synchronize()
    rs = D.RegionSort(lib, L, world, rank, types, [0, 1], [True, False], n, byte_caps, nullable=True)
    for _ in range(2):                                   # the second step reuses the regions under a new epoch
        rows, off, res = rs.step(dev, keep_result=True)
    rs.close()
    want = SR.sort_rows(full, by)
    assert SR.canon_rows(RS.rows_of(res)) == SR.canon_rows(want[off:off + rows]), "this rank's slice differs from the global order"
    top = D.RegionSort(lib, L, world, rank, types, [0, 1], [True, False], n, byte_caps, nullable=True, limit_offset=n - 7, limit_count=50)
    trows, toff, tres = top.step(dev, keep_result=True)
    top.close()
    if rank == 0:
        assert SR.canon_rows(RS.rows_of(tres)) == SR.canon_rows(SR.sort_rows(full, by, n - 7, 50)), "TopN differs from the global order"
    else:
        assert trows == 0
    counts = [None] * world
    dist.all_gather_object(counts, rows)
    assert sum(counts) == n * world
    for c in dev:
        c.free()
    print(f"DIST_SORT_OK world={world} rank={rank} rows={rows} offset={off}", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
