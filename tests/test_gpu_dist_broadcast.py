"""GPU suite: dist.BroadcastJoin across real ranks (tests/dist_broadcast_check.py) against the oracle: a string-key LEFT
OUTER join and a key-less join.  On 2 GPUs when the box has them (skipped otherwise), and always as a single rank."""
import os
import subprocess
import sys

import pytest

from test_gpu_dist import _gpu_count

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(n, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "dist_broadcast_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert f"DIST_BROADCAST_OK world={n}" in out.stdout


def test_one_rank_broadcast_join_matches_oracle():
    _run(1, 29523)


@pytest.mark.skipif(_gpu_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_broadcast_join_matches_oracle():
    _run(2, 29524)
