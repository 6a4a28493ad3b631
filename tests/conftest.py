"""pytest configuration: `gpu` marker + import paths for the oracle and the ctypes binding."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "distributed-join_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    import oracle as O

    O.build()
    return O


@pytest.fixture(scope="session")
def dj():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import djb200

    djb200.lib()  # fails loudly if the CUDA library is missing
    return djb200
