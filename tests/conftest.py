import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an NVIDIA H100 (sm_90); run with -m gpu")


@pytest.fixture(scope="session")
def po():
    """CPU oracle front-end (test infrastructure)."""
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def qcnn():
    """The product binding; the shared library must have been built (no fallback)."""
    return importlib.import_module("quantized-cnn_b200")


@pytest.fixture(scope="session")
def ctx(qcnn):
    import torch
    assert torch.cuda.is_available(), "gpu-marked test started without a GPU"
    c = qcnn.Context(0)
    yield c
    c.close()
