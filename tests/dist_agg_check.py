"""torchrun entry: dist.RegionAgg across real GPUs — a nullable two-item GROUP BY (INT64, DOUBLE with both zeros and NULLs)
against the single-process oracle on the gathered inputs, and, on a NOT NULL single key, the same groups as the NCCL path
(distributed_agg + gpu_agg_fns).  Launched by tests/test_gpu_dist_agg.py (2 ranks when 2 GPUs are visible, one rank otherwise)."""
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
    import exchange_ref as X
    import region_agg_ref as RA
    from tinysql_b200 import _lib as L
    from tinysql_b200 import dist as D
    lib = L.load()
    L.check(lib.tq_init(local))
    dev = torch.device("cuda", local)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    bm = lambda nn: t(np.concatenate([np.packbits(nn, bitorder="little"), np.zeros(16, np.uint8)]))
    I64, F64 = L.TQ_TYPE_INT64, L.TQ_TYPE_FLOAT64

    # ---- nullable multi-key
    rng = np.random.default_rng(90 + rank)
    n = 300_000 + 1000 * rank
    k1 = rng.integers(0, 5000, n).astype(np.int64)
    k2 = np.where(rng.random(n) < 0.3, -0.0 if rank % 2 else 0.0, rng.integers(0, 3, n) * 0.5)
    x = rng.integers(-4000, 4000, n) * 0.25
    nns = [rng.random(n) >= 0.05, rng.random(n) >= 0.05, rng.random(n) >= 0.05]
    types = [I64, F64, F64]
    funcs = [(COUNT, -1), (SUM, 2), (AVG, 2), (MAX, 2), (FIRSTROW, 0), (FIRSTROW, 1)]
    ra = D.RegionAgg(lib, L, world, rank, types, [0, 1], funcs, max_groups_per_rank=5000 * 4 + 16)
    torch.cuda.synchronize()
    dev_cols, dev_bms = [t(k1), t(k2), t(x)], [bm(nn) for nn in nns]
    for _ in range(2):                                   # the second step reuses the regions under a new epoch
        groups, res = ra.step(dev_cols, [b.data_ptr() for b in dev_bms], keep_result=True)
    ra.close()
    assert groups == res[0].length
    d = RA.group_dest(groups, [np.ascontiguousarray(c.values).view(np.uint64) for c in res[4:]], [c.not_null() for c in res[4:]], [False, True], world)
    assert np.all(d == rank), "a group finished on a rank its key does not name"
    gathered = [None] * world
    dist.all_gather_object(gathered, (RA.canon(res), [k1, k2, x], nns))
    if rank == 0:
        got = np.concatenate([g[0] for g in gathered])
        want = RA.oracle(types, [(g[1], g[2]) for g in gathered], [0, 1], funcs)
        assert np.array_equal(X.sorted_rows(got), RA.canon(want.cols)), "distributed nullable GROUP BY differs from the oracle"

    # ---- NOT NULL single key: RegionAgg == distributed_agg (NCCL)
    rng = np.random.default_rng(190 + rank)
    n = 400_000
    k = rng.integers(0, 100_000, n).astype(np.int64)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    funcs = [(SUM, 1), (COUNT, -1), (FIRSTROW, 0)]
    nn_types = [I64 | L.TQ_TYPE_NOT_NULL, I64 | L.TQ_TYPE_NOT_NULL]
    ra = D.RegionAgg(lib, L, world, rank, nn_types, [0], funcs, max_groups_per_rank=100_000)
    tk, tv = t(k), t(v)
    torch.cuda.synchronize()
    _, res = ra.step([tk, tv], keep_result=True)
    ra.close()
    partial_fn, final_fn = D.gpu_agg_fns(lib, L, [I64, I64], 0, funcs)
    nccl = D.distributed_agg([tk, tv], world, rank, partial_fn, D.gpu_partition_fn(lib, L), final_fn)
    assert np.array_equal(RA.canon(res), RA.canon(nccl)), "RegionAgg and distributed_agg differ"

    # ---- the int64 limits, four steps on one RegionAgg: exact; a merged total past INT64_MAX (its owner fails, the others
    # are exact); a part past INT64_MAX on one rank (every rank fails); exact again.  Every rank builds every rank's shard
    # from one seed, so each can name its own expected status and groups (region_agg_ref.expect_ranks).
    import int_agg_ref as I
    from tinysql_b200.chunk import Chunk, Column
    lfuncs = [(COUNT, -1), (SUM, 1), (AVG, 1), (FIRSTROW, 0)]
    ltypes = [I64, I64]
    frng = np.random.default_rng(77)
    fam = I.limits(frng, n_groups=200, hi=400)
    past_twin = I.out_by_one(fam, I.INT64_MAX + 1, frng)
    sizes, tot = np.bincount(fam.gid), I.group_totals(fam)
    big = max((g for g in range(len(sizes)) if tot[g] >= 0), key=lambda g: sizes[g])
    steps = [("limits", I.deal(frng, fam, world, rebuild=True)),
             ("merged_past", I.deal(frng, past_twin, world, rebuild=True)),
             ("part_past", I.deal(frng, fam, world, rebuild=True, past=(big, world - 1)) if world > 1 else I.deal(frng, past_twin, 1)),
             ("clean", I.deal(frng, fam, world, rebuild=True))]
    ra = D.RegionAgg(lib, L, world, rank, ltypes, [0], lfuncs, max_groups_per_rank=4096)
    for name, dealt in steps:
        rank_cols = [[I.key_column(d.gid) if len(d.gid) else Column(I64, np.zeros(0, np.int64), np.zeros(0, bool)), Column(I64, d.x)]
                     for d in dealt]
        exp = RA.expect_ranks(ltypes, rank_cols, [0], lfuncs, world)
        assert {"limits": not exp.push_fail and not exp.dest_fail, "clean": not exp.push_fail and not exp.dest_fail,
                "merged_past": bool(exp.push_fail) if world == 1 else (not exp.push_fail and len(exp.dest_fail) == 1),
                "part_past": bool(exp.push_fail)}[name], (name, exp.push_fail, exp.dest_fail)
        key, x = rank_cols[rank]
        dk, dx, dbm = t(key.values), t(x.values), bm(key.not_null())
        torch.cuda.synchronize()
        try:
            _, res = ra.step([dk, dx], [dbm.data_ptr(), None], keep_result=True)
            status = L.TQ_OK
        except L.TQError as e:
            status, res = e.status, None
        fails = bool(exp.push_fail) or rank in exp.dest_fail
        assert status == (L.TQ_ERR_OVERFLOW_BIGINT if fails else L.TQ_OK), (name, rank, status)
        if not fails:
            bad = I.mismatches(I.result_rows(Chunk(res), [3]), exp.ranks[rank], lfuncs)
            assert not bad, (name, rank, bad[:5])
    ra.close()
    print(f"DIST_AGG_OK world={world} rank={rank} groups={res[0].length}", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
