import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (select with -m gpu)")


def _has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built_extension():
    """The CUDA extension is built in-tree by __graft_entry__.build(); build it here too if a test run starts
    from a clean checkout (nvcc cross-compiles sm_90a without a GPU).  Tests never fall back to anything else."""
    from summerset_b200 import build as b
    b.build()
    yield


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure). Built on demand from oracle/ss_oracle.c."""
    from oracle import pyoracle
    pyoracle.build()
    pyoracle.lib()
    return pyoracle


@pytest.fixture(scope="session")
def ctx():
    """A device context on cuda:0 / torch's current stream. GPU tests only."""
    import torch
    from summerset_b200.api import Context
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    c = Context(0)
    yield c
    c.close()
