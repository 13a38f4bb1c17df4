import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")
    # the oracle (torch-CPU) runs on the threads this process may really use, not on every core of the machine
    import torch
    from oracle import usable_cpus
    torch.set_num_threads(min(usable_cpus(), 64))


@pytest.fixture(scope="session")
def built():
    """The CUDA library and the oracle are built once per session (nvcc cross-compiles without a GPU)."""
    import __graft_entry__
    __graft_entry__.build()
    return True
