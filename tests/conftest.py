import os
import sys

# the oracle's OpenMP workers must not spin between calls: on a many-core box they starve torch's own CPU side
os.environ.setdefault("OMP_WAIT_POLICY", "PASSIVE")
os.environ.setdefault("GOMP_SPINCOUNT", "0")

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    import dhqr_oracle as O
    return O


@pytest.fixture(scope="session")
def coracle(oracle):
    return oracle.COracle()
