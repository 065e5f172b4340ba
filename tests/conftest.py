import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def _engine_session():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import cpb200

    return cpb200.get_engine()


@pytest.fixture
def engine(_engine_session):
    """The process-wide engine, reset to the product default (tensor-core Gram) before every test."""
    _engine_session.gram_mode = 1
    return _engine_session
