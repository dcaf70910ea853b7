import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


@pytest.fixture(scope="session")
def built_lib():
    """Make sure the C-ABI library exists (nvcc cross-compiles without a GPU)."""
    from nvmolkit_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g

        g.build()
    return _lib.load()


@pytest.fixture(scope="session")
def cuda(built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nvmolkit_b200 import _lib

    _lib.check(built_lib.b200mol_check_device(0))
    return torch.device("cuda:0")
