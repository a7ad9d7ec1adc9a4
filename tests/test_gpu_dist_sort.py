"""GPU suite: dist.RegionSort across 2 real GPUs (tests/dist_sort_check.py) against sort_ref.  The 2-GPU run is skipped on a
box with fewer; the same script as one rank (a process group of one, every row pushed to itself) runs on any GPU box."""
import os
import subprocess
import sys

import pytest

from test_gpu_dist import _gpu_count

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(nproc, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1", "--master-port",
           str(port), os.path.join(ROOT, "tests", "dist_sort_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert out.stdout.count(f"DIST_SORT_OK world={nproc}") == nproc


@pytest.mark.skipif(_gpu_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_region_sort_matches_reference():
    _run(2, 29541)


@pytest.mark.skipif(_gpu_count() < 1, reason="needs a GPU")
def test_one_rank_region_sort_matches_reference():
    _run(1, 29542)
