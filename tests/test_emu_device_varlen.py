"""CPU suite: var-len columns from device memory into the sort / TopN and merge join (csrc/sort.cu, which also holds the
device append of var-len cells that every operator uses) run WITHOUT a GPU, under the tests/emu build (see test_emu_kernels.py): the bodies of test_gpu_zz_device_varlen.py against the
oracle.  The hash join and the aggregation are not part of the emulation build; their var-len device puts are checked by the
`-m gpu` tests only."""
import pytest

import test_gpu_zz_device_varlen as TV
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)


@pytest.mark.parametrize("n,piece", [(1, 100), (700, 150), (2500, 900)])
def test_emu_sort_string_by_items_from_device(emu, n, piece):  # noqa: F811
    TV.sort_body(emu, n, piece)


def test_emu_merge_join_string_keys_from_device(emu):  # noqa: F811
    TV.merge_join_body(emu, 600, 900)


def test_emu_device_varlen_rules(emu):  # noqa: F811
    TV.sort_mjoin_rules(emu)
