import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with `-m gpu`)")


@pytest.fixture(scope="session", autouse=True)
def _build_oracle_c():
    from oracle import march
    march.build()


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from neuralsim_b200 import _lib
    _lib.lib()  # fail loudly if the library is missing
    return torch.device("cuda:0")
