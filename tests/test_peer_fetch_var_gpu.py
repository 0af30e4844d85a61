"""NVLink pull shuffle of variable-length records: each process sorts OrderedWordCount-shaped records that it generated
on the device with sort_device (Text keys, HashPartitioner) into its exported buffer, pulls its partitions from the
others with the checksum verified in flight, and merges the pulled segments in place.  The processes share cuda:0
(CUDA IPC maps a buffer of the same device just as well), so the test runs on a one-GPU box; every owned partition must
equal the oracle's merge of the producers' oracle runs byte for byte (tests/peer_var_worker.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world,n,P", [(2, 40000, 8), (3, 10000, 7)])
def test_sort_device_pull_merge_across_processes(world, n, P):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29700 + world), os.path.join(ROOT, "tests", "peer_var_worker.py"),
           str(n), str(P), "3"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("ok") == world
