"""CPU suite: tq_partition_device (csrc/partition.cu, the multi-GPU exchange's stable radix partition) executed WITHOUT a GPU
through the emulation build of tests/emu, running the bodies of tests/test_gpu_exchange.py's section A against the exact
reference of tests/exchange_ref.py: bit-for-bit data, bitmaps and part_offsets at the warp-chunk (2048 rows) and block
(16384 rows) edges, 1..256 partitions, 1..16 columns, edge and aimed keys, scratch reuse, and the refusals.  The push paths
of join.cu use TMA and clusters and are only checked on the H100."""
import numpy as np
import pytest

import test_gpu_exchange as TX
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)

SIZES = [0, 1, 2047, 2048, 2049, 16383, 16384, 16385, 40_001]


@pytest.mark.parametrize("n", SIZES)
def test_emu_partition_matches_stable_reference(emu, n):
    TX.test_partition_matches_stable_reference(emu, n)


def test_emu_partition_edge_keys_and_skew(emu):
    TX.test_partition_edge_keys_and_skew(emu, n=5000)


def test_emu_partition_scratch_reuse(emu):
    TX.test_partition_scratch_reuse(emu, big=20000, small=3001)


def test_emu_partition_refusals(emu):
    TX.test_partition_refusals(emu)


@pytest.mark.parametrize("n_parts", [1, 2, 3, 7, 8, 64, 255, 256])
def test_emu_partition_all_null_keys(emu, n_parts):
    """every key NULL: rows go round-robin (row % n_parts), in input order within a partition"""
    rng = np.random.default_rng(n_parts)
    n = 9000
    io = TX._PartIO(emu, [rng.integers(0, 1 << 62, n).astype(np.uint64), np.arange(n, dtype=np.uint64)], [np.zeros(n, bool), None])
    try:
        TX._check_partition(emu, rng, n, n_parts, 2, 0, True, False, io=io)
        want = np.concatenate([np.arange(p, n, n_parts) for p in range(n_parts)]).astype(np.uint64)
        assert np.array_equal(io.result()[1][0], want)
    finally:
        io.free()
