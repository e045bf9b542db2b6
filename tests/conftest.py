import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture()
def cpu_context():
    import openembedding_b200 as oe
    from openembedding_b200.context import reset_context
    reset_context()
    old = oe.flags.device
    oe.flags.device = "cpu"
    yield
    reset_context()
    oe.flags.device = old


@pytest.fixture()
def cuda_context():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import openembedding_b200 as oe
    from openembedding_b200.context import reset_context
    reset_context()
    old = oe.flags.device
    oe.flags.device = "cuda"
    yield
    reset_context()
    oe.flags.device = old
