import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a)")
    config.addinivalue_line("markers", "slow: long-running CPU oracle checks")


@pytest.fixture(scope="session")
def panels():
    z = np.load(os.path.join(GOLDEN, "hom_fac_1_panels.npz"))
    return {k: z[k] for k in z.files}


@pytest.fixture(scope="session")
def notebook_tables():
    import json
    return json.load(open(os.path.join(GOLDEN, "notebook_tables.json")))
