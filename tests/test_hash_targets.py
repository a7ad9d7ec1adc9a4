"""CPU suite: tests/hash_targets.py restates the library's placement hashes and their inverses for the key-aiming edge tests
(test_gpu_hash_edges.py).  If a hash of the library changes, those tests would quietly turn back into random tests; this
check fails instead.  The library's own tqd::hash_key / tqd::mix64 come from the emulation build (tests/emu), which compiles
csrc/common.cuh with g++."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hash_targets as H

EMU_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")


@pytest.fixture(scope="module")
def product():
    subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
    lib = C.CDLL(os.path.join(EMU_DIR, "libtq_emu.so"))
    for name in ("tq_emu_hash_key", "tq_emu_mix64"):
        getattr(lib, name).restype = C.c_uint64
        getattr(lib, name).argtypes = [C.c_uint64]
    return lib


def _values():
    rng = np.random.default_rng(2024)
    edge = [0, 1, 2, 0xFFFFFFFF, 1 << 32, (1 << 32) + 1, (1 << 63) - 1, 1 << 63, (1 << 64) - 1, H.EMPTY_KEY, H.GOLDEN, 0xA5A5A5A5A5A5A5A5]
    edge += [1 << b for b in range(64)]
    return np.concatenate([np.array(edge, dtype=np.uint64), rng.integers(0, 1 << 64, 3000, dtype=np.uint64, endpoint=False)])


def test_restated_hashes_equal_the_library(product):
    v = _values()
    got_h, got_m = H.hash_key(v), H.mix64(v)
    for i, x in enumerate(v.tolist()):
        assert int(got_h[i]) == product.tq_emu_hash_key(x), hex(x)
        assert int(got_m[i]) == product.tq_emu_mix64(x), hex(x)
    # int64 bit patterns hash like their uint64 reinterpretation
    assert np.array_equal(H.hash_key(v.view(np.int64)), got_h)


def test_inverses_round_trip():
    v = _values()
    assert np.array_equal(H.hash_key_inv(H.hash_key(v)), v)
    assert np.array_equal(H.hash_key(H.hash_key_inv(v)), v)
    assert np.array_equal(H.mix64_inv(H.mix64(v)), v)
    assert np.array_equal(H.mix64(H.mix64_inv(v)), v)


def test_dist_dest_rank_uses_mix64():
    from tinysql_b200 import dist
    v = _values().view(np.int64)
    for world in (1, 2, 3, 8):
        want = ((H.mix64(v) >> np.uint64(40)) % np.uint64(world)).astype(np.int64)
        assert np.array_equal(dist.dest_rank_np(v, world), want)


def test_aimed_keys_land_where_aimed():
    rng = np.random.default_rng(5)
    for top_bits in (1, 6, 12):
        k = H.join_keys(rng, 500, (1 << top_bits) - 1, top_bits, (1 << 32) - 2048, 1 << 32, avoid_signbit=(top_bits == 6))
        h = H.hash_key(k)
        assert len(np.unique(k)) == 500 and not (k.view(np.uint64) == np.uint64(H.EMPTY_KEY)).any()
        assert (H.table_of(h, top_bits) == (1 << top_bits) - 1).all()
        for cap in (16, 4752, 33392, 1 << 20):          # the last slot whatever the capacity
            assert (H.home_slot(h, cap, 2) == cap - 1).all()
            assert (H.home_slot(h, cap, 1) == (cap - 2 if cap % 2 == 0 else cap - 1)).all()
        if top_bits == 6:
            assert (k >= 0).all()
    for r in range(1, 8):                               # r << 29: exactly the start of CTA slice r of a cluster-built sub-table
        k = H.join_keys(rng, 50, 0, 12, r << 29, (r << 29) + 1)
        for cap in (4752, 21248, 33392, 41440):
            assert (H.home_slot(H.hash_key(k), cap, 2) == r * cap // 8).all()
    k = H.agg_keys(rng, 300, 24, (1 << 24) - 1)
    for mask_bits in (16, 18, 24):
        assert ((H.mix64(k) & np.uint64((1 << mask_bits) - 1)) & ~np.uint64(3) == np.uint64((1 << mask_bits) - 4)).all()
    f = H.join_keys_not_in_tables(rng, 1000, [0, 63], 6)
    assert not np.isin(H.table_of(H.hash_key(f), 6), [0, 63]).any()


def test_restated_geometry_matches_the_documented_figures():
    # DESIGN §2 / the streaming-build change: C3 (1e7 build rows, 2 columns) -> 41,440-entry sub-tables; 3 columns -> 21,248
    g = H.stream_geometry(10_000_000, 2)
    assert g["cap"] == 41440
    g = H.stream_geometry(10_000_000, 3)
    assert (g["cap"], g["bin_slab"], g["lbits"], g["max_rows"]) == (21248, 28512, 1, 10624)
    g = H.stream_geometry(1_000_000, 2, 20000)
    assert (g["max_rows"], g["bin_slab"]) == (16696, 23648)
    assert H.stream_geometry(100_000, 2) is None
