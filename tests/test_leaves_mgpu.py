"""The leaf accessors on the replica that b200tsdf_gather_volume builds from real shards (needs >= 2 GPUs; skipped otherwise):
it must enumerate exactly like the unsharded volume, and the shards themselves must refuse (tests/mgpu_leaves_worker.py)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_gathered_replica_enumerates_like_the_whole_volume(engine_lib, oracle_lib):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29541", os.path.join(ROOT, "tests", "mgpu_leaves_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "MGPU_LEAVES_OK world=2" in r.stdout
