import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'mix-of-show_b200')
for p in (ROOT, PKG):  # PKG also exposes the top-level gradient_fusion module
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; select with -m gpu)')


@pytest.fixture(scope='session')
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    # the PyTorch references must be true fp32 (no TF32) to serve as the yardstick
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device('cuda:0')
