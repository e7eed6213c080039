import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.golden import GOLDEN, H, load_golden  # noqa: E402,F401


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def pkg():
    import paillier_b200
    return paillier_b200


@pytest.fixture(scope="session")
def cuda_engine(pkg):
    """The product engine (CUDA build).  GPU tests must run on it and nothing else."""
    eng = pkg.get_engine()
    eng.require_device()
    assert eng.path.endswith("python-paillier_b200/libpaillier_b200.so")
    return eng
