import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an sm_90a GPU; select with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """gpu-marked tests need a CUDA device: on a box without one they are skipped, not failed
    (the product itself still fails loudly there -- tests/test_host_logic.py checks that)."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Both shared objects exist before any test runs (nvcc cross-compiles without a GPU)."""
    import gaccum_b200
    assert gaccum_b200.version() >= 100      # forces the (lazy) build + load of csrc/libgaccum.so
    import oracle_c
    oracle_c.build()
    yield
