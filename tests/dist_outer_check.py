"""torchrun entry: dist.RegionJoin running a LEFT OUTER join of nullable columns with an outer-side filter across real GPUs
(masked region pushes over CUDA IPC, tq_region_gather, the local outer join), checked against the single-process oracle on
the gathered inputs.  Launched by tests/test_gpu_dist_outer.py (skipped when fewer than 2 GPUs are visible)."""
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
    from tinysql_b200 import _lib as L
    from tinysql_b200 import dist as D
    from tinysql_b200.chunk import INT64, Column
    lib = L.load()
    L.check(lib.tq_init(local))
    dev = torch.device("cuda", local)
    rng = np.random.default_rng(70 + rank)
    nb, npr = 50_000 + 1000 * rank, 200_000 + 777 * rank
    bk = rng.integers(0, 40_000, nb).astype(np.int64)                # duplicate build keys
    bv = np.arange(nb, dtype=np.int64) + rank * 10_000_000
    pk = rng.integers(0, 60_000, npr).astype(np.int64)               # a third of the probe keys have no match
    pv = np.arange(npr, dtype=np.int64) + rank * 10_000_000
    bnn, pnn = rng.random(nb) >= 0.05, rng.random(npr) >= 0.05      # NULL keys on both sides
    pvn = rng.random(npr) >= 0.2                                     # NULL payload cells
    sel = (rng.random(npr) >= 0.1).astype(np.uint8)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    bm = lambda nn: t(np.concatenate([np.packbits(nn, bitorder="little"), np.zeros(16, np.uint8)]))
    bmaps = [bm(bnn), bm(np.ones(nb, bool))]
    pmaps = [bm(pnn), bm(pvn)]
    rj = D.RegionJoin(lib, L, world, rank, 50_000 + 1000 * (world - 1), 200_000 + 777 * (world - 1), n_chunks=2, join_type=1,
                      outer_is_right=False, build_nullable=True, probe_nullable=True)
    tb, tp, ts = [t(bk), t(bv)], [t(pk), t(pv)], t(sel)
    torch.cuda.synchronize()
    for _ in range(2):                                               # the second step reuses the regions under a new epoch
        rows, _, res = rj.step_cols(tb, tp, [b.data_ptr() for b in bmaps], [p.data_ptr() for p in pmaps], ts, keep_result=True)
    rj.close()
    assert rows == (res[0].length if res else 0)
    got = np.stack([np.where(c.not_null(), c.raw(), np.uint64(0xDEAD)) for c in res], axis=1) if rows else np.zeros((0, 4), np.uint64)
    gathered = [None] * world
    dist.all_gather_object(gathered, (got, bk, bv, pk, pv, bnn, pnn, pvn, sel))
    if rank == 0:
        import oracle_py as O
        cat = lambda i: np.concatenate([g[i] for g in gathered])
        g = cat(0)
        want = O.hash_join(1, False, [INT64, INT64], [Column(INT64, cat(1), cat(5)), Column(INT64, cat(2))], [INT64, INT64],
                           [Column(INT64, cat(3), cat(6)), Column(INT64, cat(4), cat(7))], [0], [0], selected=cat(8))
        w = np.stack([np.where(c.not_null(), c.raw(), np.uint64(0xDEAD)) for c in want.cols], axis=1)
        key = lambda m: m[np.lexsort(m.T[::-1])]
        assert g.shape == w.shape, (g.shape, w.shape)
        assert np.array_equal(key(g), key(w)), "distributed LEFT OUTER join differs from the oracle"
        print(f"DIST_OUTER_OK world={world} rows={g.shape[0]}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
