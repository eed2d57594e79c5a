import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA GPU (H100); run with -m gpu")
    # emulation tests spin on real OS threads: a protocol bug must fail, not hang (marker of pytest-timeout; a no-op without it)
    config.addinivalue_line("markers", "timeout(seconds): per-test time limit (pytest-timeout)")


def _has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def native():
    """The native library must be built (python -c 'import __graft_entry__ as g; g.build()')."""
    import bevy_hanabi_b200 as hb
    return hb


@pytest.fixture()
def ctx(native):
    """A fresh simulation context on cuda:0. GPU tests fail (not skip) if the context cannot be created."""
    c = native.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="session")
def orc():
    from oracle import c_oracle
    return c_oracle.load()
