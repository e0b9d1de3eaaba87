import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def official_weights():
    """Seeded synthetic Mimi weights (oracle/mimi_spec.py); digest-checked against the fixtures."""
    import numpy as np
    from oracle import mimi_spec as S
    from oracle.gen_golden import weights_digest
    w = S.synthetic_weights(S.OFFICIAL, seed=41)
    g = np.load(os.path.join(ROOT, "tests", "golden", "mimi_cfg1.npz"))
    assert weights_digest(w) == str(g["weights_sha256"]), "synthetic weight RNG drifted from the golden fixtures"
    return w
