import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture
def oracle_ops(monkeypatch):
    """Route the product's operator surface to the plain-torch oracle so host-side logic can run on CPU.
    (Test seam only — the product itself has no such switch.)"""
    from dynamicpdb_b200 import kernels
    from oracle import ops
    for name in ops.ALL:
        monkeypatch.setattr(kernels, name, getattr(ops, name))
    return ops
