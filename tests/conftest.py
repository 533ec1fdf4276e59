import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (H100); run with -m gpu')


@pytest.fixture(scope='session')
def cuda_lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from nerf_from_image_b200 import _lib
    return _lib.load()  # raises if the extension is missing: no fallback
