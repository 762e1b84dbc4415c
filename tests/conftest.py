import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")
    config.addinivalue_line("markers", "slow: takes about a minute of host CPU (full-size oracle)")


@pytest.fixture(scope="session")
def built():
    """Build libape_b200.so + the oracle once per session (no-op when up to date)."""
    import __graft_entry__ as g

    g.build()
    return True


def load_golden(name):
    import numpy as np
    import torch

    z = np.load(os.path.join(GOLDEN, name))
    return {k: torch.from_numpy(z[k]) for k in z.files}
