"""torchrun entry: dist.RegionAgg across real GPUs on device string columns — GROUP BY a nullable VARCHAR with SUM, COUNT(*),
MAX / MIN of the same column and FIRSTROW, over two steps that reuse the regions — against the single-process oracle on the
gathered inputs.  Launched by tests/test_gpu_dist_agg_strings.py (2 ranks when 2 GPUs are visible, one rank otherwise)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COUNT, SUM, AVG, MAX, MIN, FIRSTROW = range(6)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    import region_agg_strings_ref as S
    from tinysql_b200 import _lib as L
    from tinysql_b200 import dist as D
    from tinysql_b200.chunk import BYTES, Column, VarColumn
    lib = L.load()
    L.check(lib.tq_init(local))
    I64 = L.TQ_TYPE_INT64

    rng = np.random.default_rng(300 + rank)
    n = 200_000
    words = [b""] + [b"key-%06d" % i for i in range(20_000)]
    s = VarColumn(BYTES, [None if rng.random() < 0.02 else words[i] for i in rng.integers(0, len(words), n)])
    x = Column(I64, rng.integers(-1000, 1000, n).astype(np.int64), rng.random(n) >= 0.05)
    types, funcs = [BYTES, I64], [(SUM, 1), (COUNT, -1), (MAX, 0), (MIN, 0), (FIRSTROW, 0)]
    caps = [int(s.offsets[-1]) + 1, None]
    gathered_caps = [None] * world
    dist.all_gather_object(gathered_caps, caps[0])
    caps[0] = max(gathered_caps)                          # every rank passes the same numbers: the layout is shared
    ra = D.RegionAgg(lib, L, world, rank, types, [0], funcs, max_groups_per_rank=len(words) + 1, byte_caps=caps)
    dev = S.device([s, x])
    torch.cuda.synchronize()
    for _ in range(2):                                   # the second step reuses the regions under a new epoch
        groups, res = ra.step(dev, keep_result=True)
    ra.close()
    for c in dev:
        c.free()
    assert groups == res[0].length
    assert np.all(S.dest_of(res[4:], types, [0], world) == rank), "a group finished on a rank its key does not name"
    gathered = [None] * world
    dist.all_gather_object(gathered, (S.rows_of(res), [s.tolist(), x.values, x.not_null()]))
    if rank == 0:
        got = sorted([r for g in gathered for r in g[0]], key=lambda r: tuple((v is None, repr(v)) for v in r))
        shards = [[VarColumn(BYTES, g[1][0]), Column(I64, g[1][1], g[1][2])] for g in gathered]
        assert got == S.rows_of(S.oracle(types, shards, [0], funcs)), "distributed string GROUP BY differs from the oracle"
    print(f"DIST_AGG_STRINGS_OK world={world} rank={rank} groups={groups}", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
