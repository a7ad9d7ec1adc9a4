"""CPU suite: the kernels of csrc/sort.cu (radix sort, gathers, merge-join search / expand) and csrc/codec.cu (k_chunk_unpack)
executed WITHOUT a GPU.  tests/emu compiles those product sources unchanged with g++ against an emulation of the CUDA primitives
they use (one OS thread per CUDA thread, pthread barriers for __syncthreads and the warp collectives — tests/emu/include/
cuda_runtime.h) into libtq_emu.so, which exports the same C-ABI entry points.  The host-side mirror (tinysql_b200/executor.py,
chunk.py) is pointed at that library and the bodies of the GPU parity tests run against the oracle.  This checks the code's
LOGIC (indexing, ranking, masks, searches, the host orchestration); timing, memory-model and launch behaviour are what the
`-m gpu` tests of the same names check on the H100."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import test_gpu_chunk_codec as TC
import test_gpu_sort_merge as TS
import test_gpu_string_filter as TF
import test_gpu_zz_device_chain as TD
from sort_cases import MERGE_CASES, SORT_CASES
from tinysql_b200 import _lib as L

EMU_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
EMU_SO = os.path.join(EMU_DIR, "libtq_emu.so")


@pytest.fixture(scope="module")
def emu_lib():
    subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
    lib = C.CDLL(EMU_SO)
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = res, args
    return lib


@pytest.fixture()
def emu(emu_lib, monkeypatch):
    monkeypatch.setattr(L, "_lib", emu_lib)   # executor.py / chunk.py call L.load()
    return emu_lib


@pytest.mark.parametrize("case", SORT_CASES, ids=[c[0] for c in SORT_CASES])
def test_emu_sort_reference_goldens(emu, case):
    TS.test_sort_reference_goldens(emu, case)


@pytest.mark.parametrize("case", MERGE_CASES, ids=[c[0] for c in MERGE_CASES])
def test_emu_merge_join_reference_goldens(emu, case):
    TS.test_merge_join_reference_goldens(emu, case)


@pytest.mark.parametrize("n", [0, 1, 2, 255, 256, 257, 4095, 4096, 4097, 9001])
def test_emu_sort_every_layout_vs_oracle(emu, n):
    TS.test_sort_every_layout_vs_oracle(emu, n)


def test_emu_sort_wide_keys_and_long_strings(emu, monkeypatch):
    TS.test_sort_wide_keys_and_long_strings(emu, n=3000)


@pytest.mark.parametrize("jt,oir", [(0, False), (1, False), (2, True)])
def test_emu_merge_join_vs_oracle(emu, jt, oir):
    TS.test_merge_join_vs_oracle(emu, jt, oir, ni=3000, no=5000)


def test_emu_merge_join_typed_keys_default_inner_and_unsorted_input(emu):
    TS.test_merge_join_typed_keys_default_inner_and_unsorted_input(emu)


def test_emu_chunk_decode_golden(emu):
    TC.test_reference_test_codec_golden_on_device(emu)


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 63, 64, 65, 1000, 10003])
@pytest.mark.parametrize("null_frac", [0.0, 0.3])
def test_emu_chunk_decode_equals_host_decode(emu, n, null_frac):
    TC.test_device_decode_equals_host_decode(emu, n, null_frac)


def test_emu_chunk_decode_rejects_truncated_buffers(emu):
    TC.test_device_decode_rejects_truncated_buffers(emu)


def test_emu_string_filter_reference_vectors(emu):
    TF.test_reference_vectors(emu)
    TF.test_error_of_the_last_non_null_row(emu)


@pytest.mark.parametrize("seed", range(4))
def test_emu_string_filter_differential_fuzz(emu, seed):
    TF.test_differential_fuzz(emu, seed, n=6000)


@pytest.mark.parametrize("jt,oir", [(0, False), (1, False), (2, True), (0, True)])
def test_emu_merge_join_other_conditions(emu, jt, oir):
    TS.test_merge_join_other_conditions(emu, jt, oir, ni=2000, no=3000)


@pytest.mark.parametrize("n,piece", [(0, 1000), (1, 1000), (5001, 900), (5001, 100000)])
def test_emu_sort_device_chunks(emu, n, piece):
    TD.test_sort_device_chunks(emu, n, piece)


def test_emu_device_chunk_rules(emu):
    TD.test_device_chunk_rules(emu)


def test_emu_sort_sort_merge_join_chain_on_the_device(emu):
    """the chain of test_join_then_sort_then_merge_join_stay_on_the_device with the oracle standing in for the hash join
    (join.cu is not part of the emulation build): its result is uploaded as the producer's device columns"""
    import oracle_py as O
    from tinysql_b200.chunk import DeviceColumn
    types, b, p = TD.chain_tables(3000, 20000)
    want_join = O.hash_join(0, True, types, b, types, p, [0], [0])
    dj = [DeviceColumn.from_host(c) for c in want_join.cols]
    TD.chain_after_join(emu, TD.arr_nn(dj), lambda: [d.free() for d in dj], want_join, types, b)
