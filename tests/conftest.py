import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90); run with -m gpu on a machine that has one")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    d = os.path.join(ROOT, "tests", "golden")
    return {k: np.load(os.path.join(d, f"{k}.npz")) for k in ("scenario_1", "scenario_2", "scenario_3", "hudson_bay")}


@pytest.fixture(scope="session")
def O():
    """The CPU oracle (test infrastructure)."""
    from oracle import oracle
    oracle.build()
    return oracle
