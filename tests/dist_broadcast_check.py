"""torchrun entry: dist.BroadcastJoin across real GPUs (broadcast pushes over CUDA IPC, one device build chunk per source,
the local probe shard), checked against the single-process oracle on the gathered inputs: a LEFT OUTER join on a BIGINT +
VARCHAR key with NULLs, selected[] and string payloads, then a key-less join with ON b.x < p.x, whose rank outputs in rank
order are the oracle's exact sequence.  Launched by tests/test_gpu_dist_broadcast.py on 2 GPUs (when visible) and as a
single rank."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _strings(rng, n, lo, hi, null_frac):
    nn = rng.random(n) >= null_frac
    return [b"k%05d" % v if ok else None for v, ok in zip(rng.integers(lo, hi, n), nn)], nn


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    from tinysql_b200 import _lib as L
    from tinysql_b200 import dist as D
    from tinysql_b200.chunk import BYTES, INT64, Chunk, Column, DeviceColumn
    lib = L.load()
    L.check(lib.tq_init(local))
    rng = np.random.default_rng(90 + rank)
    nb, npr = 20_000 + 500 * rank, 60_000 + 333 * rank
    s, snn = _strings(rng, nb, 0, 300, 0.05)
    build = [Column(INT64, rng.integers(0, 40, nb), rng.random(nb) >= 0.05), Column(BYTES, s, snn), Column(BYTES, [b"b%d" % i for i in range(nb)])]
    s, snn = _strings(rng, npr, 0, 400, 0.05)
    probe = [Column(INT64, rng.integers(0, 50, npr), rng.random(npr) >= 0.05), Column(BYTES, s, snn), Column(INT64, np.arange(npr) + rank * 10**7)]
    sel = rng.random(npr) >= 0.1
    bt, pt = [INT64, BYTES, BYTES], [INT64, BYTES, INT64]
    caps = [None, 8 * (20_000 + 500 * (world - 1)), 8 * (20_000 + 500 * (world - 1))]
    dev = lambda cols: [DeviceColumn.from_host(c) for c in cols]
    db, dp = dev(build), dev(probe)
    bj = D.BroadcastJoin(lib, L, world, rank, 20_000 + 500 * (world - 1), bt, pt, [0, 1], [0, 1], join_type=1, outer_is_right=False,
                         byte_caps=caps, build_nullable=True, probe_nullable=True)
    for _ in range(2):                                               # the second step reuses the regions under a new epoch
        rows, _, keyed = bj.step_cols(db, dp, selected=sel, keep_result=True)
    assert rows == keyed[0].length
    bj.close()
    # key-less: ON b.x < p.x over left = probe ++ right = build (outer_is_right = 0), inner join
    kb, kp = [Column(INT64, rng.integers(0, 100, 300))], [Column(INT64, rng.integers(0, 100, 500)), Column(INT64, np.arange(500))]
    dkb, dkp = dev(kb), dev(kp)
    bk = D.BroadcastJoin(lib, L, world, rank, 300, [INT64], [INT64, INT64], join_type=0, outer_is_right=False, other_conditions=[(0, 2, 0)])
    _, _, keyless = bk.step_cols(dkb, dkp, keep_result=True)
    bk.close()
    for d in db + dp + dkb + dkp:
        d.free()
    gathered = [None] * world
    dist.all_gather_object(gathered, (keyed, build, probe, sel, keyless, kb, kp))
    if rank == 0:
        import oracle_py as O
        from keyless_oracle import keyless_hash_join
        from util import assert_same_multiset, assert_same_ordered
        cat = lambda i, types: Chunk.concat([Chunk(g[i]) for g in gathered], types).cols
        want = O.hash_join(1, False, bt, cat(1, bt), pt, cat(2, pt), [0, 1], [0, 1], np.concatenate([g[3] for g in gathered]))
        got = Chunk.concat([Chunk(g[0]) for g in gathered], pt + bt)
        assert_same_multiset(got, want)
        kall = cat(5, [INT64])
        for r in range(world):
            assert_same_ordered(Chunk(gathered[r][4]), keyless_hash_join(0, False, [INT64], kall, [INT64, INT64], gathered[r][6], conds=[(0, 2, 0)]))
        print(f"DIST_BROADCAST_OK world={world} rows={got.num_rows()}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
