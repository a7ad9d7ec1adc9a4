"""GPU suite: dist.RegionJoin's LEFT OUTER join of nullable columns across 2 real GPUs (tests/dist_outer_check.py) against
the oracle.  Needs >= 2 GPUs on the box; skipped otherwise."""
import os
import subprocess
import sys

import pytest

from test_gpu_dist import _gpu_count

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(_gpu_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_left_outer_region_join_matches_oracle():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29519",
           os.path.join(ROOT, "tests", "dist_outer_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "DIST_OUTER_OK world=2" in out.stdout
