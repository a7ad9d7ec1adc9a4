"""CPU suite: the merge-join cases of test_gpu_join_program.py (OtherConditions as an expression program, csrc/sort.cu k_mj_prog
and the interpreter of csrc/expr_prog.cuh) run against the emulation build of tests/emu, as test_emu_kernels.py does for the
other merge-join cases.  The hash join (join.cu) is not part of the emulation build; its cases run on the GPU only."""
import pytest

import test_gpu_join_program as TJ
from test_emu_kernels import emu, emu_lib  # noqa: F401  (fixtures)
from test_oracle_join_program import out_types
from join_program_oracle import conds_to_program
from tinysql_b200.chunk import INT64, UINT64
from util import assert_same_ordered


@pytest.mark.parametrize("jt,oir", TJ.JOINS)
def test_emu_merge_join_program_vs_oracle(emu, jt, oir):
    TJ.test_merge_join_program_vs_oracle(emu, jt, oir, ni=2000, no=3000)


@pytest.mark.parametrize("jt,oir", [(0, False), (1, False), (2, True)])
def test_emu_merge_join_overflow_raises_only_for_evaluated_rows(emu, jt, oir):
    TJ.test_overflow_raises_only_for_evaluated_rows(emu, "merge", jt, oir)


def test_emu_merge_join_abi_rejections(emu):
    TJ.test_abi_rejections(emu, "merge")


@pytest.mark.parametrize("jt,oir", TJ.JOINS)
def test_emu_merge_join_program_form_equals_comparison_form(emu, jt, oir):
    import numpy as np
    t = TJ.make_tables(np.random.default_rng(jt + 2 * int(oir)), oir, 2000, 3000, sort=True)
    p = t.pos
    for conds in ([(0, p["is"], p["ov"])], [(3, p["id"], p["od"]), (5, p["iu"], None, UINT64, 7), (1, p["iv"], None, INT64, 0)]):
        a, _ = TJ.run("merge", jt, oir, t.it, t.ic, t.ot, t.oc, [0], [1], conds=conds)
        b, _ = TJ.run("merge", jt, oir, t.it, t.ic, t.ot, t.oc, [0], [1], conds_to_program(conds, out_types(oir, t.it, t.ot)))
        assert_same_ordered(a, b)
