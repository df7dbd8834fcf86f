import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests', 'golden')):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')

try:  # torch reference ops must be true fp32 (cuDNN/cuBLAS default to TF32 for convs)
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
except Exception:  # pragma: no cover
    pass


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: test needs a CUDA device (run on an H100 with -m gpu)')


@pytest.fixture(scope='session')
def golden_dir():
    return GOLDEN
