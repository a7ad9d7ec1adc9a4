"""CPU suite: the sort / TopN / merge-join edge families of test_gpu_sort_edges.py run WITHOUT a GPU, under the tests/emu build
(see test_emu_kernels.py), against the exact reference of tests/sort_ref.py: orders, TopN windows, digit-pass counts and the
merge join's refusals.  The emulation compiles scan.cu, so the result-size guard of a merge join whose emit counts pass 2^32
inside one scan tile (4096 outer rows x (2^20 + 1) inner rows) runs through the product's scan here too; the 2^26-row
result and the second guard shape are `-m gpu` only."""
import pytest

import test_gpu_sort_edges as TE
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)


@pytest.mark.parametrize("case", TE.SORTS, ids=[c.name for c in TE.SORTS])
def test_emu_sort_family(emu, case):  # noqa: F811
    TE.sort_family_body(emu, case)


def test_emu_sort_refuses_more_than_eight_by_items(emu):  # noqa: F811
    TE.too_many_by_items_body(emu)


@pytest.mark.parametrize("case", TE.MJS, ids=[c.name for c in TE.MJS])
def test_emu_merge_join_family(emu, case):  # noqa: F811
    TE.mj_family_body(emu, case)


@pytest.mark.parametrize("with_conds", [False, True])
def test_emu_merge_join_result_past_2_32_rows_in_one_scan_tile_is_refused(emu, with_conds):  # noqa: F811
    TE.size_guard_body("i", with_conds)
