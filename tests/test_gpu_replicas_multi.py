"""The replica step across ranks: W = 2 ranks x 2 replicas against W = 1 x 4 replicas under neg = 0
(tests/replica_multi_worker.py).  With neg = 0 no row is drawn at random, so the per-rank losses sum to the gathered
loss and the all-reduced gradients equal the one-process gradients; with neg > 0 they differ only in neg_filter's keep
ratio, taken per rank's shard.  Runs on two GPUs with NCCL, or on one GPU with both ranks and gloo."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_ranks_of_two_replicas_equal_one_rank_of_four():
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node=2',
           os.path.join(ROOT, 'tests', 'replica_multi_worker.py')]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    print('\n'.join(l for l in r.stdout.splitlines() if 'REPLICA_MULTI_OK' in l))
    assert r.returncode == 0 and r.stdout.count('REPLICA_MULTI_OK') == 2, r.stdout[-6000:]
