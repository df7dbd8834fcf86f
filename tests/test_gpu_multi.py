"""Multi-GPU data parallelism on real devices (needs >= 2 GPUs; skipped on one GPU).  The host-side
bucket logic has its CPU twin in tests/test_distributed_cpu.py (gloo, world size 2)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_rank_allreduce_equals_sum_of_shards_and_graph_step_matches_eager():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr', '127.0.0.1',
           '--master-port', '29611', os.path.join(ROOT, 'tests', 'multi_gpu_worker.py')]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=240)
    assert r.returncode == 0 and r.stdout.count('MULTI_OK') == 2, r.stdout[-4000:]
