"""A total-order sort across processes: each of G processes sharing cuda:0 generates records on the device, the
processes agree on split points sampled on the device (shuffle.total_order_splits), sort with TotalOrderPartitioner,
pull their blocks of partitions through CUDA IPC with the checksum verified in flight and merge them in place.  Every
owned partition must equal the oracle's merge of the producers' oracle runs byte for byte, so rank 0's output, then
rank 1's, ... is the oracle's sort of all records (tests/total_order_sort_worker.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world,n,P,kind", [(2, 30000, 8, "bytes"), (3, 20000, 7, "words"), (2, 20000, 16, "words")])
def test_total_order_sort_across_processes(world, n, P, kind):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    port = 29740 + world + (10 if kind == "words" else 0) + P
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "total_order_sort_worker.py"),
           str(n), str(P), kind]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("ok") == world
